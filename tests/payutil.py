"""Shared by the payload tests and scripts/microbench_index.py --payloads: term-major lists whose hits carry payloads, shaped to reach the
encoders' edges, the reference's SegmentIndexSession fed payloads (tref_index_documents_payloads, oracle/ref_indexer_payloads.cpp), and a numpy
model of the inversion that carries them.  TEST INFRASTRUCTURE ONLY — never imported by the product package."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

from idxutil import term_order

ROOT = Path(__file__).resolve().parent.parent
SO = ROOT / "oracle" / "_ref" / "libtrinity_ref_indexer_payloads.so"
MAX_POSITION = 1 << 14
_lib = None


def load_indexer_payloads():
    global _lib
    if _lib is None:
        if not SO.exists():
            subprocess.check_call(["bash", str(ROOT / "oracle" / "build_indexer_payloads.sh")])
        L = C.CDLL(str(SO))
        L.tidxp_last_error.restype = C.c_char_p
        L.tidxp_last_ms.restype = C.c_double
        L.tref_index_documents_payloads.argtypes = [C.c_int, C.c_char_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, C.c_void_p, C.c_uint32]
        _lib = L
    return _lib


def masked(sizes, vals):
    """the payloads with the bytes past each size cleared (what a reader hands back)"""
    sizes = np.asarray(sizes, np.uint8)
    m = np.array([(1 << (8 * int(x))) - 1 if x < 8 else (1 << 64) - 1 for x in sizes], np.uint64)
    return np.asarray(vals, np.uint64) & m


def term(rng, ndocs, freq_of, size_of, max_gap=50, span=MAX_POSITION, first=0, pos0=False):
    """one term: ndocs ascending docIDs, freq_of(i) hits of document i at sorted random positions (pos0: a document's first hit at 0),
    size_of(i, k) the payload size of hit k of document i; payloads random 64-bit values with the bytes past the size set too (a
    reader must not see them)"""
    docs = (first + np.cumsum(rng.integers(1, max_gap, ndocs, dtype=np.uint64))).astype(np.uint32)
    freqs = np.array([freq_of(i) for i in range(ndocs)], np.uint32)
    pos, sz = [], []
    for i, f in enumerate(freqs.tolist()):
        p = np.sort(rng.integers(1, span, f)).astype(np.uint32)
        if pos0 and f:
            p[0] = 0
        pos.append(p)
        sz.extend(size_of(i, k) for k in range(f))
    pos = np.concatenate(pos).astype(np.uint32) if pos else np.zeros(0, np.uint32)
    sz = np.array(sz, np.uint8)
    if pos0:
        first_hit = np.r_[0, np.cumsum(freqs)[:-1]][freqs > 0].astype(np.int64)
        sz[first_hit] = np.maximum(sz[first_hit], 1)  # a position-0 hit needs a payload
    vals = rng.integers(0, 1 << 63, size=len(pos), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=len(pos), dtype=np.uint64)
    return docs, freqs, pos, sz, vals


def five_byte_term(rng):
    """docID deltas >= 2^28 (5-byte codes), a 17 000-hit document (3-byte freq) whose sizes change at random"""
    docs = np.array([7, 7 + (1 << 28) + 3, 7 + (1 << 29), 4_000_000_000], np.uint32)
    freqs = np.array([1, 2, 17_000, 1], np.uint32)
    pos = np.concatenate([[MAX_POSITION - 1], [5, 9000], np.sort(rng.integers(1, MAX_POSITION, 17_000)), [3]]).astype(np.uint32)
    sz = rng.integers(0, 9, size=len(pos)).astype(np.uint8)
    vals = rng.integers(0, 1 << 63, size=len(pos), dtype=np.uint64)
    return docs, freqs, pos, sz, vals


def google_shapes(rng):
    """(name, term) pairs: every size 0..8, a change at every hit / at no hit / only at document starts, position-0 payload hits,
    5-byte varbyte codes and a 17 000-hit document, enough blocks for skiplist entries and a countdown carried across terms"""
    return [
        ("every-size", term(rng, 40, lambda i: 1 + i % 5, lambda i, k: (i * 5 + k) % 9)),
        ("change-every-hit", term(rng, 33, lambda i: 4, lambda i, k: 1 + (k % 2) * 6)),
        ("no-change", term(rng, 70, lambda i: 1 + i % 3, lambda i, k: 0)),
        ("doc-starts-only", term(rng, 65, lambda i: 1 + i % 4, lambda i, k: 1 + i % 8)),
        ("pos0", term(rng, 50, lambda i: 1 + i % 3, lambda i, k: (i + k) % 9, pos0=True)),
        ("freq-0-docs", term(rng, 35, lambda i: i % 2 * 3, lambda i, k: 8)),
        ("skiplist", term(rng, 32 * 21 + 5, lambda i: 1 + (i * 7) % 4, lambda i, k: (i // 3) % 9, max_gap=300)),
        ("5-byte", five_byte_term(rng)),
        ("tail", term(rng, 3, lambda i: 2, lambda i, k: 2 + k)),
    ]


def lucene_shapes(rng):
    """(name, term) pairs for the LUCENE layout: payload-size int-blocks in every PFor form (all 0, all equal, mostly 0 with a few
    8s as exceptions, mixed), full hit blocks spanning documents, tails whose size changes across documents, hits ending exactly at
    a 128-hit boundary"""
    few8 = lambda i, k: 8 if (i * 3 + k) % 41 == 0 else 0  # noqa: E731
    return [
        ("sizes-all-0", term(rng, 200, lambda i: 1 + i % 3, lambda i, k: 0)),
        ("sizes-all-3", term(rng, 200, lambda i: 1 + i % 3, lambda i, k: 3)),
        ("sizes-few-8", term(rng, 300, lambda i: 1 + i % 4, few8)),
        ("sizes-mixed", term(rng, 150, lambda i: 1 + i % 5, lambda i, k: (i * 7 + k * 3) % 9)),
        ("spanning", term(rng, 6, lambda i: 90 + 17 * i, lambda i, k: (k // 20) % 9, span=4000)),
        ("tail-changes", term(rng, 9, lambda i: 5, lambda i, k: i % 3 * 2)),
        ("at-boundary", term(rng, 64, lambda i: 4, lambda i, k: (i + k) % 9)),  # 256 hits: two full blocks, an empty tail
        ("pos0", term(rng, 140, lambda i: 1 + i % 2, lambda i, k: 1 + k, pos0=True)),
        ("5-byte", five_byte_term(rng)),
        ("no-hits", term(rng, 4, lambda i: 0, lambda i, k: 0)),
    ]


def ref_index_payloads(codec, path, names, docids, offs, tok, pos, plens, payloads):
    """the reference's SegmentIndexSession over the batch with payloads, fed in docID order (as idxutil.ref_index_flat does), committed
    into `path`; returns its host ms"""
    L = load_indexer_payloads()
    f = L.tref_index_documents_payloads
    Path(path).mkdir(parents=True, exist_ok=True)
    docids, offs, tok = np.asarray(docids, np.uint32), np.asarray(offs, np.uint64), np.asarray(tok, np.uint32)
    pos = None if pos is None else np.asarray(pos, np.uint32)
    plens, payloads = np.asarray(plens, np.uint8), np.asarray(payloads, np.uint64)
    by_id = np.argsort(docids, kind="stable")
    lens = np.diff(offs).astype(np.int64)
    new = np.r_[0, np.cumsum(lens[by_id])].astype(np.int64)
    gather = np.repeat(offs[:-1].astype(np.int64)[by_id] - new[:-1], lens[by_id]) + np.arange(len(tok), dtype=np.int64)
    tok, plens, payloads = tok[gather], plens[gather], payloads[gather]
    pos = None if pos is None else pos[gather]
    docids, offs = docids[by_id], new.astype(np.uint64)
    enc = [n.encode() for n in names]
    arr = (C.c_char_p * len(enc))(*enc)
    p = lambda a: None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)  # noqa: E731
    keep = [np.ascontiguousarray(x) for x in (docids, offs, tok, plens, payloads)] + ([np.ascontiguousarray(pos)] if pos is not None else [])
    rc = f(codec, str(path).encode(), C.cast(arr, C.c_void_p), len(enc), p(keep[0]), p(keep[1]), p(keep[2]), p(keep[5]) if pos is not None else None,
           p(keep[3]), p(keep[4]), len(docids))
    if rc != 0:
        raise RuntimeError(L.tidxp_last_error().decode())
    return float(L.tidxp_last_ms())


def model_postings_payloads(docids, offs, tok, pos, plens, payloads, nterms):
    """the inversion in numpy with payloads: [(term id, (docids, freqs, positions, sizes, payloads))] in index order (equal positions of a
    term in a document keep their token order: the tests give them equal payloads)"""
    lens = np.diff(np.asarray(offs, np.uint64)).astype(np.int64)
    doc = np.repeat(np.asarray(docids, np.int64), lens)
    pos = (np.concatenate([np.arange(1, n + 1) for n in lens]) if pos is None else np.asarray(pos)).astype(np.int64)
    place = np.empty(nterms, np.int64)
    place[term_order(nterms)] = np.arange(nterms)
    tok = np.asarray(tok, np.int64)
    o = np.lexsort((pos, doc, place[tok]))
    t, d, p, sz, pv = tok[o], doc[o], pos[o], np.asarray(plens, np.uint8)[o], masked(plens, payloads)[o]
    out = []
    tb = np.flatnonzero(np.r_[True, t[1:] != t[:-1], True]) if len(t) else np.zeros(1, np.int64)
    for a, b in zip(tb[:-1], tb[1:]):
        dd = d[a:b]
        pb = np.flatnonzero(np.r_[True, dd[1:] != dd[:-1], True])
        out.append((int(t[a]), (dd[pb[:-1]].astype(np.uint32), np.diff(pb).astype(np.uint32), p[a:b].astype(np.uint32), sz[a:b], pv[a:b])))
    return out


def zipf_payloads(rng, ntok):
    """random payload sizes 0..8 and bytes for ntok tokens"""
    return rng.integers(0, 9, size=ntok).astype(np.uint8), rng.integers(0, 1 << 63, size=ntok, dtype=np.uint64) * np.uint64(2)
