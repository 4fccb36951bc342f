"""The compact result stream, word for word: every segment of every (query, tile) work item of the tile-emitting routes of k_exec_docs
equals a numpy restatement of the encodings of include/trinity_b200.h (trn_result), computed from the reference's docIDs:
  * the encoding rule: bitmap unless fewer words suffice; 16-bit offsets; bucketed 8-bit offsets for tiles of 2^13 docIDs or more whose
    256-docID buckets all hold fewer than 256 documents;
  * the bytes: U8B count bytes, offset bytes and zero pad bytes; U16 offsets and the zero pad half-word; bitmap words.
Routes: all-bitmap run tickets, flat ANDs with some and with no bitmap operands, flat OR, flat tree, step programs (a GOOGLE phrase and
every LUCENE plan).  Also the plain DocumentsOnly stream, masked documents, TRN_DOCS_SHIFT 13/14/15, TRN_TREE_SHIFT 12/13, and the top tile
of the docID space by translation (as test_gpu_docid_limits)."""
import ctypes as C
import os

import numpy as np
import pytest

import trinity_b200 as tb
from refharness import RefIndex

pytestmark = pytest.mark.gpu

G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE
S = 600_000
TOP = 2**32 - 2
DELTA = TOP - S
ENC = {"u32": 0, "u16": 1, "bitmap": 2, "u8b": 3}  # item_desc >> 30 (TRN_ENC_*)
FULL = np.arange(204_800, 205_056, dtype=np.uint32)  # one whole 256-docID bucket (aligned in the 2^13 .. 2^15 tiles holding it)


def _corpus():
    u = lambda *a: np.unique(np.concatenate([np.asarray(x, np.uint32) for x in a]))
    out = {}
    for name, step in (("a", 2), ("b", 3), ("c", 5), ("d", 7), ("e", 11)):  # dense: a resident bitmap each
        out[name] = np.arange(step, S + 1, step, dtype=np.uint32)
    out["f"] = u(np.arange(6, S + 1, 6), FULL, [S])  # dense, with the full bucket: "f AND g" holds 256 documents there
    out["g"] = u(np.arange(7, S + 1, 7), FULL - 100, FULL, FULL + 100, [S])
    out["m"] = np.arange(37, S + 1, 37, dtype=np.uint32)  # decoded terms
    out["p"] = np.arange(41, S + 1, 41, dtype=np.uint32)
    out["h"] = u(np.arange(40, S + 1, 40), np.arange(S - 3000, S + 1))  # no bitmap; "h AND k": 1 in 40, and a full top
    out["k"] = u(np.arange(40, S + 1, 40), np.arange(23, S + 1, 1009), np.arange(S - 3000, S + 1))
    out["s"] = np.arange(401, S + 1, 401, dtype=np.uint32)
    return out


LISTS = _corpus()
NAMES = list(LISTS)
# query -> the route it takes on GOOGLE (LUCENE: step programs)
QUERIES = {
    "a AND b": tb.ROUTE_FLAT_AND,  # all-bitmap: bitmap tiles (1 in 6)
    "a AND e": tb.ROUTE_FLAT_AND,  # all-bitmap: U8B (1 in 22)
    "c AND d AND e": tb.ROUTE_FLAT_AND,  # all-bitmap: U16 (1 in 385)
    "f AND g": tb.ROUTE_FLAT_AND,  # all-bitmap: the full bucket
    "b AND c AND f": tb.ROUTE_FLAT_AND,  # all-bitmap, odd counts
    "c AND m": tb.ROUTE_FLAT_AND,  # one bitmap operand
    "h AND k": tb.ROUTE_FLAT_AND,  # no bitmap operand: U8B, bitmap in the top tiles
    "m AND p": tb.ROUTE_FLAT_AND,  # no bitmap operand: U16
    "m OR p OR s": tb.ROUTE_FLAT_OR,
    "a OR m": tb.ROUTE_FLAT_OR,
    "(a OR m) AND (b OR s) NOT e": tb.ROUTE_FLAT_TREE,
    "(h AND m) OR (p AND k)": tb.ROUTE_FLAT_TREE,
}
PHRASE = '"c d"'  # GOOGLE: a step program (in a batch of its own: a batch with a phrase plan does not take the run tickets)


def _positions(name, d):
    """c's only hit sits at position 1, d's at position 2 (phrase "c d" matches where both are present); the rest: 1 .. freq"""
    return {"c": np.ones(len(d), np.uint32), "d": np.full(len(d), 2, np.uint32)}.get(name)


def _freqs(name, d):
    return np.ones(len(d), np.uint32) if name in ("c", "d") else (1 + d % 3).astype(np.uint32)


def _index(codec, shift):
    b = tb.IndexBuilder(codec)
    for n in NAMES:
        d = LISTS[n]
        b.add_term((d.astype(np.uint64) + shift).astype(np.uint32), _freqs(n, d), _positions(n, d))
    return b.index(), b.terms_array()


@pytest.fixture(scope="module")
def refidx(ref):
    out = {}
    for codec in (G, L):
        r = RefIndex(ref, codec)
        for n in NAMES:
            r.add_term(n, LISTS[n], _freqs(n, LISTS[n]), _positions(n, LISTS[n]))
        r.finish(S)
        out[codec] = r
    return out


def _source(codec, shift, max_docid, env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        g = tb.GpuIndexSource(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k)
            else:
                os.environ[k] = v
    g.upload(codec, *_index(codec, shift), max_docid)
    return g


def _expected_segment(docs, first, shift):
    """(encoding, words) of a tile's documents as the rule picks them; docs: sorted uint64 docIDs of the tile"""
    W, n = 1 << shift, len(docs)
    NW = W >> 5
    rel = (docs - first).astype(np.int64)
    nbk = W >> 8
    full = n and np.bincount(rel >> 8, minlength=nbk).max() >= 256
    enc, words = ENC["bitmap"], NW
    if W <= 65536:
        if (n + 1) // 2 < words:
            enc, words = ENC["u16"], (n + 1) // 2
        if NW >= 256 and not full and (nbk + n + 3) // 4 < words:
            enc, words = ENC["u8b"], (nbk + n + 3) // 4
    if enc == ENC["bitmap"]:
        out = np.zeros(NW, np.uint32)
        np.bitwise_or.at(out, rel >> 5, (np.uint32(1) << (rel & 31).astype(np.uint32)))
    elif enc == ENC["u16"]:
        h = np.zeros(2 * words, np.uint16)
        h[:n] = rel
        out = h.view("<u4")
    else:
        b = np.zeros(4 * words, np.uint8)
        b[:nbk] = np.bincount(rel >> 8, minlength=nbk)
        b[nbk: nbk + n] = rel & 255
        out = b.view("<u4")
    return enc, out



class QItems(C.Structure):
    _fields_ = [("item_base", C.c_uint32), ("nitems", C.c_uint32), ("tile_lo", C.c_uint32), ("tile_shift", C.c_uint32)]


def _check_stream(res, wants, qs, seen):
    """every segment of every query of a copy=False MODE_DOCS_COMPACT result against _expected_segment; seen collects the encodings and
    the special cases met"""
    raw = res.raw
    nq = res.nq
    off = np.ctypeslib.as_array(raw.offsets, shape=(nq + 1,))
    words = np.ctypeslib.as_array(raw.words, shape=(max(int(raw.total_words), 1),))
    desc = np.ctypeslib.as_array(raw.item_desc, shape=(max(res.nitems, 1),))
    qi = C.cast(raw.qitems, C.POINTER(QItems))
    for q in range(nq):
        want = wants[q].astype(np.uint64)
        Q = qi[q]
        w, at = int(off[q]), 0
        for j in range(Q.nitems):
            d = int(desc[Q.item_base + j])
            n, enc = d & 0x3FFFFFFF, d >> 30
            first = (Q.tile_lo + j) << Q.tile_shift
            lo_i, hi_i = np.searchsorted(want, [first, first + (1 << Q.tile_shift)])
            docs = want[lo_i:hi_i]
            assert n == len(docs), f"[{qs[q]}] item {j}: {n} documents, the reference has {len(docs)}"
            if not n:
                continue
            at += n
            xenc, xw = _expected_segment(docs, first, Q.tile_shift)
            assert enc == xenc, f"[{qs[q]}] item {j} (tile {first:#x}, {n} documents): encoding {enc}, the rule gives {xenc}"
            got = words[w: w + len(xw)]
            assert np.array_equal(got, xw), f"[{qs[q]}] item {j} (tile {first:#x}, encoding {enc}): {np.flatnonzero(got != xw)[:8]} differ"
            w += len(xw)
            seen.add(("enc", enc, Q.tile_shift))
            rel = docs - first
            if enc == ENC["u8b"] and (((1 << Q.tile_shift) >> 8) + n) % 4:
                seen.add("u8b pad")
            if enc == ENC["u16"] and n % 2:
                seen.add("u16 pad")
            if len(rel) and np.bincount((rel >> 8).astype(np.int64)).max() >= 256 and enc != ENC["bitmap"]:
                seen.add("full bucket")
        assert at == len(want), f"[{qs[q]}] the items hold {at} documents, the reference {len(want)}"
        assert w == int(off[q + 1]), f"[{qs[q]}] the segments take {w - int(off[q])} words, the query {int(off[q + 1] - off[q])}"


def _run(refidx, codec, shift, max_docid, env, masked=None):
    """both DocumentsOnly modes of the queries (GOOGLE: and the phrase, in a batch of its own) on a fresh source; returns what
    _check_stream saw"""
    batches = [list(QUERIES)] + ([[PHRASE]] if codec == G else [])
    g = _source(codec, shift, max_docid, env)
    seen = set()
    try:
        if masked is not None:
            g.set_masked_documents((masked.astype(np.uint64) + shift).astype(np.uint32))
        tdict = tb.TermDictionary(NAMES)
        r = refidx[codec]
        for qs in batches:
            plans = [tb.parse_query(q, tdict) for q in qs]
            wants = [(r.exec(q, False, S + 1)[0] if masked is None else r.exec_masked(q, False, masked, S + 1)[0]).astype(np.uint64) + shift
                     for q in qs]
            plain = g.exec_batch(plans, tb.MODE_DOCS_ONLY)
            routes = list(g.last_routes())
            for i, q in enumerate(qs):
                assert np.array_equal(plain.query(i)[0].astype(np.uint64), wants[i]), f"[{q}] plain DocumentsOnly stream"
            comp = g.exec_batch(plans, tb.MODE_DOCS_COMPACT, copy=False)
            assert list(g.last_routes()) == routes
            exp = [QUERIES.get(q, tb.ROUTE_STEPS) if codec == G else tb.ROUTE_STEPS for q in qs]
            assert routes == exp, (qs, routes, exp)
            _check_stream(comp, wants, qs, seen)
    finally:
        g.close()
    return seen


@pytest.mark.parametrize("docs_shift", [13, 14, 15])
def test_stream_google(refidx, docs_shift):
    env = {"TRN_DOCS_SHIFT": str(docs_shift), "TRN_TREE_SHIFT": "12" if docs_shift == 13 else "13"}
    index, terms = _index(G, 0)
    plans = [tb.parse_query(q, tb.TermDictionary(NAMES)) for q in QUERIES]
    _, tickets = tb.debug_dense_runs(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=S)
    assert {0, 1, 2, 3, 4} <= set(tickets[:, 0].tolist())  # the all-bitmap ANDs run on the run tickets
    seen = _run(refidx, G, 0, S, env)
    for enc in ("bitmap", "u16", "u8b"):
        assert ("enc", ENC[enc], docs_shift) in seen, (enc, seen)
    assert {"u8b pad", "u16 pad", "full bucket"} <= seen, seen
    assert any(x[2] == int(env["TRN_TREE_SHIFT"]) for x in seen if isinstance(x, tuple)), seen  # the flat-tree launch's tiles


def test_stream_lucene(refidx):
    seen = _run(refidx, L, 0, S, {})
    for enc in ("bitmap", "u16", "u8b"):
        assert ("enc", ENC[enc], 14) in seen, (enc, seen)


def test_stream_masked(refidx):
    rng = np.random.default_rng(21)
    pool = np.unique(np.concatenate([LISTS["a"][::4], LISTS["f"][::3], LISTS["h"][-2000:], LISTS["m"][::2], FULL[::7]]))
    masked = np.sort(rng.choice(pool, size=len(pool) // 2, replace=False)).astype(np.uint32)
    for codec in (G, L):
        _run(refidx, codec, 0, S, {}, masked)


@pytest.mark.parametrize("codec", [G, L], ids=["google", "lucene"])
def test_stream_top_of_the_docid_space(refidx, codec):
    seen = _run(refidx, codec, DELTA, TOP, {})
    assert ("enc", ENC["bitmap"], 14) in seen
