"""GPU-side Encoder for the LUCENE layout (trn_encode_lucene == Codecs::Lucene::Encoder, lucene_codec.cpp:163-388): the index and its
hits.data built on the device are BYTE-IDENTICAL to what this repo's host encoder writes for the same postings (term tuples included), and
equal to the reference encoder's bytes wherever the reference does not leave PFor padding uninitialised.  Covered: terms of 0 / 1 / 127 /
128 / 129 / 256 / 128*9+77 documents, all-equal int-blocks, freq-0 documents, PFor exceptions with maxb - b == 1 and >= 2 up to 32-bit
values, 5-byte varbyte tail deltas, hits that fill whole 128-hit blocks, a document with 17 000 hits, 2- and 3-byte tail position codes,
the 65 535-entry skiplist cap, refused inputs, and an encoded index executed against the reference's exec_query."""
import ctypes as C

import numpy as np
import pytest

import trinity_b200 as tb
from refharness import RefIndex
from util import assert_same_docs, assert_topk_equal

pytestmark = pytest.mark.gpu

MAX_POSITION = 1 << 14  # Trinity::Limits::MaxPosition (trinity_limits.h:15)


def _positions(rng, freqs, span=MAX_POSITION):
    pos = [np.sort(rng.integers(1, span, int(f))) for f in freqs]
    return np.concatenate(pos).astype(np.uint32) if pos else np.zeros(0, np.uint32)


def _term(rng, n, max_gap, freq_of, span=MAX_POSITION):
    docs = np.cumsum(rng.integers(1, max_gap, n, dtype=np.uint64)).astype(np.uint32) if n else np.zeros(0, np.uint32)
    freqs = np.array([freq_of(i) for i in range(n)], np.uint32)
    return docs, freqs, _positions(rng, freqs, span)


def _outliers(rng, n, small, big, every):
    """docID gaps below `small` with a gap near `big` every `every` documents: PFor exceptions of a chosen width"""
    gaps = rng.integers(1, small, n, dtype=np.uint64)
    gaps[::every] = big + rng.integers(0, big // 4 + 1, len(gaps[::every]))
    docs = np.cumsum(gaps).astype(np.uint32)
    freqs = (1 + rng.integers(0, 3, n)).astype(np.uint32)
    return docs, freqs, _positions(rng, freqs)


def _shapes():
    rng = np.random.default_rng(2024)
    top = np.uint32(0xFFFFFFFE)
    wide = np.concatenate([np.arange(1, 128, dtype=np.uint32), [top]]).astype(np.uint32)  # delta >= 2^31 in a full block: maxb = 32
    wide_f = np.ones(128, np.uint32)
    five = np.array([7, 7 + (1 << 28) + 3, 7 + (1 << 29), 4_000_000_000], np.uint32)       # 5-byte varbyte tail deltas
    five_f = np.array([1, 2, 17_000, 1], np.uint32)                                         # a document with 17 000 hits (3-byte freq)
    five_p = np.concatenate([[MAX_POSITION - 1], [5, 9000], np.sort(rng.integers(1, MAX_POSITION, 17_000)), [3]]).astype(np.uint32)
    const_d = (np.arange(1, 5 * 128 + 1, dtype=np.uint32) * 3).astype(np.uint32)          # all-equal doc, freq and hit int-blocks
    const_f = np.full(5 * 128, 2, np.uint32)
    const_p = np.tile(np.array([5, 10], np.uint32), 5 * 128)
    tailpos_d = np.array([10, 20, 30, 40], np.uint32)                                        # tail position codes of 1, 2 and 3 bytes
    tailpos_f = np.array([1, 1, 2, 1], np.uint32)
    tailpos_p = np.array([40, 100, 9000, 16_000, 16_383], np.uint32)
    return [
        ("empty", _term(rng, 0, 50, lambda i: 0)),
        ("one", _term(rng, 1, 50, lambda i: 3)),
        ("127", _term(rng, 127, 40, lambda i: 1 + i % 3)),
        ("128", _term(rng, 128, 40, lambda i: 1 + i % 4)),
        ("129", _term(rng, 129, 40, lambda i: 2)),
        ("256", _term(rng, 256, 300, lambda i: 1 + (i * 7) % 5)),
        ("9x128+77", _term(rng, 128 * 9 + 77, 1000, lambda i: 1 + (i % 11 == 0) * 6)),
        ("constant", (const_d, const_f, const_p)),
        ("freq-0", _term(rng, 128 * 3 + 5, 20, lambda i: i % 3)),
        ("exc-k1", _outliers(rng, 128 * 4, 8, 12, 9)),                 # outliers one bit wider than the rest
        ("exc-k>=2", _outliers(rng, 128 * 4, 16, 1 << 20, 17)),        # outliers many bits wider
        ("32-bit", (wide, wide_f, np.arange(1, 129, dtype=np.uint32) % 7 + 1)),
        ("empty-again", _term(rng, 0, 50, lambda i: 0)),
        ("hits-128n", _term(rng, 64, 30, lambda i: 4)),                # 256 hits: no hit tail
        ("5-byte", (five, five_f, five_p)),
        ("tail-positions", (tailpos_d, tailpos_f, tailpos_p)),
        ("wide-gaps", _term(rng, 700, 3_000_000, lambda i: 1 + i % 2)),
    ]


def _best_b(v):
    """FastPFor<4>::getBestBFromData (fastpfor.h:143-171) -> (b, maxb); None for an all-equal block"""
    v = [int(x) for x in v]
    if all(x == v[0] for x in v):
        return None
    hist = [0] * 33
    for x in v:
        hist[x.bit_length()] += 1
    maxb = max(x.bit_length() for x in v)
    best, bestcost, c = maxb, maxb * 128, 0
    for bb in range(maxb - 1, -1, -1):
        c += hist[bb + 1]
        cost = c * 8 + c * (maxb - bb) + bb * 128 + 8 - (c if maxb - bb == 1 else 0)
        if cost < bestcost:
            best, bestcost = bb, cost
    return best, maxb


def _host(lists):
    b = tb.IndexBuilder(tb.CODEC_LUCENE)
    for d, f, p in lists:
        b.add_term(d, f, p)
    return b.index(), b.hits(), b.terms_array()


def _first_diff(a, b):
    d = np.flatnonzero(a[: min(a.size, b.size)] != b[: min(a.size, b.size)])
    return int(d[0]) if d.size else min(a.size, b.size)


def test_the_shapes_cover_every_int_block_form():
    kinds = set()
    for _, (d, f, p) in _shapes():
        deltas = np.diff(np.concatenate([[0], d.astype(np.int64)]))
        for j in range(len(d) // 128):
            for blk in (deltas[128 * j:128 * j + 128], f[128 * j:128 * j + 128]):
                r = _best_b(blk)
                kinds.add("equal" if r is None else ("k=0" if r[0] == r[1] else "k=1" if r[1] - r[0] == 1 else "k>=2"))
                if r is not None and r[1] == 32:
                    kinds.add("32-bit")
    assert kinds >= {"equal", "k=0", "k=1", "k>=2", "32-bit"}, kinds


@pytest.mark.parametrize("with_positions", [True, False], ids=["positions", "no-positions"])
def test_device_encoder_equals_the_host_encoder(with_positions):
    lists = [(d, f, p if with_positions else None) for _, (d, f, p) in _shapes()]
    want_i, want_h, want_t = _host(lists)
    g = tb.GpuIndexSource(0)
    index, hits, terms, ms = g.encode_lucene(lists)
    assert index.size == want_i.size and np.array_equal(index, want_i), f"index: first differing byte at {_first_diff(index, want_i)}"
    assert hits.size == want_h.size and np.array_equal(hits, want_h), f"hits.data: first differing byte at {_first_diff(hits, want_h)}"
    assert np.array_equal(terms, want_t)
    assert ms > 0
    g.close()


def test_device_encoder_equals_the_reference_encoder(ref):
    shapes = _shapes()
    r = RefIndex(ref, tb.CODEC_LUCENE)
    for name, (d, f, p) in shapes:
        r.add_term(name, d, f, p)
    r.finish(int(max(int(d.max()) if d.size else 0 for _, (d, f, p) in shapes)))
    g = tb.GpuIndexSource(0)
    index, hits, terms, _ = g.encode_lucene([l for _, l in shapes])
    assert np.array_equal(terms, r.terms())
    for mine, theirs, what in ((index, r.index(), "index"), (hits, r.hits(), "hits.data")):
        assert mine.size == theirs.size, what
        diff = np.flatnonzero(mine != theirs)
        # the reference leaves the padding of the PFor byte container uninitialised (codecs.cpp:195): only there, and only zeros of ours
        assert np.all(mine[diff] == 0), f"{what} differs at non-padding bytes {diff[:10]}"
    g.close()


def test_skiplist_is_capped_at_65535_entries():
    n = 65_536 * 128 + 5
    rng = np.random.default_rng(8)
    d = np.cumsum(rng.integers(1, 4, n, dtype=np.uint64)).astype(np.uint32)
    f = (1 + (np.arange(n) % 3 == 0)).astype(np.uint32)
    lists = [(np.array([3], np.uint32), np.array([1], np.uint32), None), (d, f, None)]
    want_i, want_h, want_t = _host(lists)
    g = tb.GpuIndexSource(0)
    index, hits, terms, _ = g.encode_lucene(lists)
    assert np.array_equal(terms, want_t)
    assert index.size == want_i.size and np.array_equal(index, want_i), f"first differing byte at {_first_diff(index, want_i)}"
    assert np.array_equal(hits, want_h)
    off = int(terms["chunk_off"][1])
    assert int(index[off + 12]) | int(index[off + 13]) << 8 == 65_535
    g.close()


def test_bad_input_is_refused():
    g = tb.GpuIndexSource(0)
    one = np.ones(4, np.uint32)
    for d, f, p in [
        (np.array([0, 3], np.uint32), one[:2], None),                                    # docID 0
        (np.array([5, 9, 9, 12], np.uint32), one, None),                                 # not ascending
        (np.array([3, 4], np.uint32), np.array([1, 1], np.uint32), np.array([0, 2], np.uint32)),  # position 0
        (np.array([3, 4], np.uint32), np.array([2, 1], np.uint32), np.array([7, 5, 1], np.uint32)),  # decreasing in a document
        (np.array([3], np.uint32), np.array([1], np.uint32), np.array([MAX_POSITION], np.uint32)),  # Limits::MaxPosition
    ]:
        with pytest.raises(tb.TrinityError, match="rc=-1"):
            g.encode_lucene([(np.array([1, 2], np.uint32), np.array([1, 1], np.uint32), None if p is None else np.array([1, 1], np.uint32)),
                             (d, f, p)])
    # a bad position inside a full 128-hit block, and a bad docID inside a full 128-document block
    d = np.arange(1, 301, dtype=np.uint32)
    f = np.ones(300, np.uint32)
    p = np.ones(300, np.uint32)
    p[70] = 0
    with pytest.raises(tb.TrinityError, match="rc=-1"):
        g.encode_lucene([(d, f, p)])
    d2 = d.copy()
    d2[60] = d2[59]
    with pytest.raises(tb.TrinityError, match="rc=-1"):
        g.encode_lucene([(d2, f, None)])
    # undersized buffers: TRN_ERR_CAPACITY with both sizes reported
    lists = [(d, f * 3, None)]
    want_i, want_h, _ = _host(lists)
    tbeg = np.array([0, 300], np.uint64)
    f3 = f * 3
    terms = np.zeros(1, dtype=tb._ffi.TERM_DTYPE)
    ib, hb, ms = C.c_uint64(), C.c_uint64(), C.c_float()
    for icap, hcap in ((want_i.size - 1, want_h.size), (want_i.size, want_h.size - 1)):
        io, ho = np.zeros(want_i.size, np.uint8), np.zeros(want_h.size, np.uint8)
        rc = g._L.trn_encode_lucene(g._h, tb._ptr(tbeg), 1, tb._ptr(d), tb._ptr(f3), None, tb._ptr(io), icap, C.byref(ib), tb._ptr(ho), hcap,
                                    C.byref(hb), tb._ptr(terms), C.byref(ms))
        assert rc == -6  # TRN_ERR_CAPACITY
        assert (ib.value, hb.value) == (want_i.size, want_h.size)
    g.close()


def test_an_index_encoded_on_the_device_executes_like_the_reference(ref):
    """encode on the GPU -> upload -> upload_hits -> exec: the judge is the reference's exec_query over the index ITS encoder wrote"""
    ndocs, nterms = 300_000, 24
    lists, names = [], []
    for rank in range(1, nterms + 1):
        d, f = tb.SynthIndex.postings(ndocs, rank, 500, 11)
        p = tb.SynthIndex.positions(ndocs, rank, 500, 11)
        lists.append((d, f, p))
        names.append(f"t{rank:04d}")
    r = RefIndex(ref, tb.CODEC_LUCENE)
    for n, (d, f, p) in zip(names, lists):
        r.add_term(n, d, f, p)
    r.finish(ndocs)
    g = tb.GpuIndexSource(0)
    index, hits, terms, _ = g.encode_lucene(lists)
    assert np.array_equal(terms, r.terms())
    for mine, theirs in ((index, r.index()), (hits, r.hits())):
        assert mine.size == theirs.size and np.all(mine[mine != theirs] == 0)
    g.upload(tb.CODEC_LUCENE, index, terms, ndocs)
    g.upload_hits(index, hits)
    tdict = tb.TermDictionary(names)
    qs = ["t0001 AND t0002", "t0003 OR t0017 OR t0024", "t0002 NOT t0005", "(t0001 OR t0009) AND (t0004 OR t0020) NOT t0003",
          '"t0001 t0002"', '"t0003 t0001 t0002"', 't0004 AND "t0001 t0002"']
    res = g.exec_batch([tb.parse_query(q, tdict) for q in qs], tb.MODE_DOCS_ONLY)
    for i, q in enumerate(qs):
        assert_same_docs(res.query(i)[0], r.exec(q, False, ndocs + 1)[0], q)
    q = "t0002 OR t0006 OR t0011 OR t0019"
    top = g.exec_batch([g.set_bm25_weights(tb.parse_query(q, tdict), ndocs)], tb.MODE_SCORED_TOPK, k=50)
    assert int(g.last_routes()[0]) == tb.ROUTE_SCORE_FLAT
    wd, ws = r.exec(q, True, ndocs + 1)
    td, ts = top.query(0)
    assert int(top.match_counts[0]) == len(wd)
    assert_topk_equal(td, ts, wd, ws, 50, f"[{q}] top-50")
    g.close()
