"""Shared by the indexer tests and scripts/microbench_index.py: the reference's SegmentIndexSession behind a C ABI
(oracle/_ref/libtrinity_ref_indexer.so, oracle/ref_indexer.cpp), corpora, and a numpy model of the doc-major -> term-major inversion.
TEST INFRASTRUCTURE ONLY — never imported by the product package."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
SO = ROOT / "oracle" / "_ref" / "libtrinity_ref_indexer.so"
FILES = ("index", "hits.data", "terms.data", "terms.idx", "id", "updated_documents.ids")
_lib = None


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def load_indexer():
    global _lib
    if _lib is None:
        if not SO.exists():
            subprocess.check_call(["bash", str(ROOT / "oracle" / "build_indexer.sh")])
        L = C.CDLL(str(SO))
        L.tidx_last_error.restype = C.c_char_p
        L.tidx_last_ms.restype = C.c_double
        L.tref_index_documents.argtypes = [C.c_int, C.c_char_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                           C.c_void_p, C.c_void_p, C.c_uint32]
        _lib = L
    return _lib


def flat(docs):
    """(doc_offsets uint64[ndocs + 1], tokens uint32[]) of a list of token arrays"""
    offs = np.zeros(len(docs) + 1, np.uint64)
    offs[1:] = np.cumsum([len(d) for d in docs])
    tok = np.concatenate([np.asarray(d, np.uint32) for d in docs]).astype(np.uint32) if len(docs) else np.zeros(0, np.uint32)
    return offs, np.ascontiguousarray(tok)


def ref_index_flat(codec, path, names, docids, offs, tok, pos=None, replaced=(), erased=()):
    """the reference's SegmentIndexSession over the batch, committed into `path` (created; its name must be a number); returns its host ms"""
    L = load_indexer()
    Path(path).mkdir(parents=True, exist_ok=True)
    # The session is fed in docID order: its duplicate tracker (SparseFixedBitSet::try_set behind consider_update, indexer.cpp:187-222) reports
    # some documents that arrive out of docID order as "Already committed".  commit() sorts the (term, document) records by docID
    # (indexer.cpp:402-410), so what it writes does not depend on the order the documents arrived in.
    docids, offs, tok = np.asarray(docids, np.uint32), np.asarray(offs, np.uint64), np.asarray(tok, np.uint32)
    by_id = np.argsort(docids, kind="stable")
    if not np.array_equal(by_id, np.arange(len(docids))):
        lens = np.diff(offs).astype(np.int64)
        new = np.r_[0, np.cumsum(lens[by_id])].astype(np.int64)
        gather = np.repeat(offs[:-1].astype(np.int64)[by_id] - new[:-1], lens[by_id]) + np.arange(len(tok), dtype=np.int64)
        tok, pos = tok[gather], (None if pos is None else np.asarray(pos, np.uint32)[gather])
        docids, offs = docids[by_id], new.astype(np.uint64)
    enc = [n.encode() if isinstance(n, str) else n for n in names]
    arr = (C.c_char_p * len(enc))(*enc)
    d = np.ascontiguousarray(docids, np.uint32)
    flags = np.isin(d, np.asarray(list(replaced), np.uint32)).astype(np.uint8) if len(replaced) else None
    er = np.ascontiguousarray(list(erased), np.uint32)
    rc = L.tref_index_documents(codec, str(path).encode(), C.cast(arr, C.c_void_p), len(enc), _p(d), _p(np.ascontiguousarray(offs, np.uint64)),
                                _p(np.ascontiguousarray(tok, np.uint32)), _p(None if pos is None else np.ascontiguousarray(pos, np.uint32)), len(d),
                                _p(flags), _p(er) if len(er) else None, len(er))
    if rc != 0:
        raise RuntimeError(L.tidx_last_error().decode())
    return float(L.tidx_last_ms())


def ref_index(codec, path, names, docids, docs, positions=None, replaced=(), erased=()):
    offs, tok = flat(docs)
    pos = None if positions is None else flat(positions)[1]
    return ref_index_flat(codec, path, names, docids, offs, tok, pos, replaced, erased)


def read_dir(path):
    """{file name: bytes} of the segment files present in a directory"""
    out = {}
    for f in FILES:
        p = Path(path) / f
        if p.exists():
            out[f] = np.fromfile(p, np.uint8)
    return out


def term_names(n, prefix="t"):
    return [f"{prefix}{i}" for i in range(n)]


def term_order(nterms):
    """order[k] = the term id at place k of the index file: commit() encodes bucket (id & 31) after bucket, ascending transient id (t + 1)
    inside a bucket (indexer.cpp:388, 402-410, 423)"""
    t = np.arange(nterms, dtype=np.int64)
    return np.lexsort((t, (t + 1) & 31))


def model_postings(docids, docs, nterms, positions=None):
    """the inversion in numpy: [(term id, docids, freqs, positions)] of the terms that have postings, in index order"""
    offs, tok = flat(docs)
    lens = np.diff(offs).astype(np.int64)
    doc = np.repeat(np.asarray(docids, np.int64), lens)
    if positions is None:
        pos = np.concatenate([np.arange(1, n + 1) for n in lens]).astype(np.int64) if len(lens) else np.zeros(0, np.int64)
    else:
        pos = flat(positions)[1].astype(np.int64)
    place = np.empty(nterms, np.int64)
    place[term_order(nterms)] = np.arange(nterms)
    o = np.lexsort((pos, doc, place[tok.astype(np.int64)]))
    t, d, p = tok[o].astype(np.int64), doc[o], pos[o]
    out = []
    tb = np.flatnonzero(np.r_[True, t[1:] != t[:-1], True]) if len(t) else np.zeros(1, np.int64)
    for a, b in zip(tb[:-1], tb[1:]):
        dd = d[a:b]
        pb = np.flatnonzero(np.r_[True, dd[1:] != dd[:-1], True])
        out.append((int(t[a]), dd[pb[:-1]].astype(np.uint32), np.diff(pb).astype(np.uint32), p[a:b].astype(np.uint32)))
    return out


def host_build(codec, model, nterms):
    """the host encoder (IndexBuilder.add_term) over the model's postings, in index order: (index, hits, terms by term id)"""
    import trinity_b200 as tb
    from trinity_b200._ffi import TERM_DTYPE

    b = tb.IndexBuilder(codec)
    terms = np.zeros(nterms, TERM_DTYPE)
    for t, d, f, p in model:
        terms[t] = b.add_term(d, f, p)
    return b.index().copy(), b.hits().copy(), terms


def zipf_corpus(ndocs, nterms, length, seed):
    """documents of `length` tokens whose terms are drawn by Zipf(1) rank over nterms terms (the percolator microbenchmark's documents):
    (docids 1 .. ndocs shuffled, doc_offsets, tokens)"""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, nterms + 1)
    cdf = np.cumsum(w / w.sum())
    tok = np.minimum(np.searchsorted(cdf, rng.random(ndocs * length)), nterms - 1).astype(np.uint32)
    offs = (np.arange(ndocs + 1, dtype=np.uint64) * np.uint64(length)).astype(np.uint64)
    docids = rng.permutation(np.arange(1, ndocs + 1, dtype=np.uint32))
    return docids, offs, tok
