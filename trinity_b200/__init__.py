"""trinity_b200 — GPU-native (H100, sm_90a) execution engine for Trinity's inverted-index hot path.

Thin Python plumbing over the C ABI (include/trinity_b200.h).  Class and method names follow the reference's
domain vocabulary (IndexSession/Encoder, IndexSource, exec_query, term_index_ctx, postings, docsets);
all decode / docset / scoring work happens in the sm_90a kernels of libtrinity_b200.so — there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Iterable, List, Optional, Sequence

import numpy as np

from ._ffi import QNODE_DTYPE, TERM_DTYPE, TrnIndexInfo, TrnQuery, TrnResult, TrnTerm, TrnTimings, lib

CODEC_GOOGLE, CODEC_LUCENE = 0, 1
MODE_DOCS_ONLY, MODE_SCORED_ALL, MODE_SCORED_TOPK = 0, 1, 2  # == ExecFlags::DocumentsOnly / AccumulatedScoreScheme (+ fused top-k sink)
MODE_DOCS_COMPACT = 3  # DocumentsOnly, compact result segments (bitmap / bucketed 8-bit offsets / 16-bit offsets / docIDs per tile): trn_result_decode replays them
NODE_TERM, NODE_AND, NODE_OR, NODE_NOT, NODE_OPTIONAL, NODE_SOME, NODE_PHRASE = 0, 1, 2, 3, 4, 5, 6
# the path a query ran (GpuIndexSource.last_routes, == TRN_ROUTE_* of include/trinity_b200.h)
ROUTE_STEPS, ROUTE_FLAT_AND, ROUTE_FLAT_OR, ROUTE_CANDIDATE, ROUTE_SCORE_FLAT, ROUTE_FLAT_TREE, ROUTE_EXEC_TILES = 0, 1, 2, 3, 4, 5, 6
EMPTY_TERM = 0xFFFFFFFF
DOC_IDS_END = 0xFFFFFFFF  # DocIDsEND, common.h:43


class TrinityError(RuntimeError):
    pass


def _u32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.uint32)


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


# ----------------------------------------------------------------------------------------------- index build (host)
class IndexBuilder:
    """== Codecs::IndexSession + Codecs::Encoder (codecs.h:66-200).  Bytes are identical to the reference encoders'."""

    def __init__(self, codec: int):
        self._L = lib()
        self.codec = codec
        h = C.c_void_p()
        if self._L.trn_builder_create(codec, C.byref(h)) != 0:
            raise TrinityError("trn_builder_create failed")
        self._h = h
        self.terms: List[tuple] = []

    def _ck(self, rc):
        if rc != 0:
            raise TrinityError(self._L.trn_builder_last_error(self._h).decode())

    def set_google_block(self, block_docs: int, skiplist_step: int = 8):
        """decode sweep only: documents per block / blocks per skiplist entry of the GOOGLE format (reference: 32 / 8)"""
        self._ck(self._L.trn_builder_set_google_block(self._h, block_docs, skiplist_step))

    def set_google_skiplist_countdown(self, n: int):
        self._ck(self._L.trn_builder_set_google_skiplist_countdown(self._h, n))

    def begin_term(self):
        self._ck(self._L.trn_builder_begin_term(self._h))

    def begin_document(self, docid: int):
        self._ck(self._L.trn_builder_begin_document(self._h, docid))

    def new_hit(self, position: int, payload: bytes = b""):
        buf = (C.c_uint8 * len(payload)).from_buffer_copy(payload) if payload else None
        self._ck(self._L.trn_builder_new_hit(self._h, position, buf, len(payload)))

    def end_document(self):
        self._ck(self._L.trn_builder_end_document(self._h))

    def end_term(self) -> tuple:
        t = TrnTerm()
        self._ck(self._L.trn_builder_end_term(self._h, C.byref(t)))
        self.terms.append((t.documents, t.chunk_off, t.chunk_len))
        return self.terms[-1]

    def add_term(self, docids, freqs, positions=None) -> tuple:
        d, f = _u32(docids), _u32(freqs)
        p = None if positions is None else _u32(positions)
        t = TrnTerm()
        self._ck(self._L.trn_builder_add_term(self._h, _ptr(d), _ptr(f), len(d), _ptr(p), C.byref(t)))
        self.terms.append((t.documents, t.chunk_off, t.chunk_len))
        return self.terms[-1]

    def _bytes(self, fn) -> np.ndarray:
        p, n = C.c_void_p(), C.c_uint64()
        self._ck(fn(self._h, C.byref(p), C.byref(n)))
        if n.value == 0:
            return np.zeros(0, dtype=np.uint8)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n.value,)).copy()

    def index(self) -> np.ndarray:
        return self._bytes(self._L.trn_builder_index)

    def hits(self) -> np.ndarray:
        return self._bytes(self._L.trn_builder_hits)

    def terms_array(self) -> np.ndarray:
        return np.array(self.terms, dtype=TERM_DTYPE)

    def __del__(self):
        try:
            self._L.trn_builder_destroy(self._h)
        except Exception:
            pass


class SynthIndex:
    """The BASELINE.md synthetic Zipfian index (SURVEY.md 8d), built multi-threaded through the host encoders."""

    def __init__(self, codec: int, ndocs: int, nterms: int = 4096, min_df: int = 1000, seed: int = 0x5EED,
                 with_hits: bool = True, threads: int = 0, doc_range: Optional[tuple] = None, google_block_docs: int = 32,
                 google_skiplist_step: int = 8):
        self._L = lib()
        self.codec, self.ndocs, self.nterms, self.min_df, self.seed = codec, ndocs, nterms, min_df, seed
        self.doc_range = doc_range or (1, ndocs)
        h = C.c_void_p()
        rc = self._L.trn_synth_build_ex(codec, ndocs, nterms, min_df, seed, int(with_hits), threads, self.doc_range[0], self.doc_range[1],
                                        google_block_docs, google_skiplist_step, C.byref(h))  # (32, 8) == the reference format
        if rc != 0:
            raise TrinityError(f"trn_synth_build failed rc={rc}")
        self._h = h
        p, n = C.c_void_p(), C.c_uint64()
        self._L.trn_synth_index(h, C.byref(p), C.byref(n))
        self.index = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n.value,))
        self._L.trn_synth_hits(h, C.byref(p), C.byref(n))
        self.hits = (np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n.value,)) if n.value
                     else np.zeros(0, dtype=np.uint8))
        tp, tn = C.c_void_p(), C.c_uint32()
        self._L.trn_synth_terms(h, C.byref(tp), C.byref(tn))
        raw = np.ctypeslib.as_array(C.cast(tp, C.POINTER(C.c_uint8)), shape=(tn.value * 12,))
        self.terms = raw.view(TERM_DTYPE)
        self.sum_hits = int(self._L.trn_synth_sum_hits(h))
        self.names = [f"t{r:04d}" for r in range(1, nterms + 1)]

    @staticmethod
    def postings(ndocs: int, rank: int, min_df: int = 1000, seed: int = 0x5EED):
        L = lib()
        n = C.c_uint32()
        L.trn_synth_postings(ndocs, rank, min_df, seed, None, None, 0, C.byref(n))
        d, f = np.zeros(n.value, np.uint32), np.zeros(n.value, np.uint32)
        L.trn_synth_postings(ndocs, rank, min_df, seed, _ptr(d), _ptr(f), n.value, C.byref(n))
        return d, f

    @staticmethod
    def positions(ndocs: int, rank: int, min_df: int = 1000, seed: int = 0x5EED):
        L = lib()
        n = C.c_uint64()
        L.trn_synth_positions(ndocs, rank, min_df, seed, None, 0, C.byref(n))
        p = np.zeros(n.value, np.uint32)
        L.trn_synth_positions(ndocs, rank, min_df, seed, _ptr(p), n.value, C.byref(n))
        return p

    def __del__(self):
        try:
            self._L.trn_synth_destroy(self._h)
        except Exception:
            pass


# ----------------------------------------------------------------------------------------------- query front-end
class TermDictionary:
    """term name -> term id; the host-side stand-in for IndexSource::resolve_term_ctx (index_source.h:118)."""

    def __init__(self, names: Sequence[str]):
        self._L = lib()
        self.names = list(names)
        enc = [s.encode("utf-8", "surrogateescape") for s in self.names]
        arr = (C.c_char_p * len(enc))(*enc)
        h = C.c_void_p()
        if self._L.trn_dict_create(C.cast(arr, C.c_void_p), len(enc), C.byref(h)) != 0:
            raise TrinityError("trn_dict_create failed")
        self._h = h  # an explicit dictionary handle: the names are copied, nothing is keyed on caller memory

    def __len__(self):
        return len(self.names)

    def __del__(self):
        try:
            self._L.trn_dict_destroy(self._h)
        except Exception:
            pass


def parse_query(text: str, tdict: TermDictionary, min_match: Optional[int] = None) -> np.ndarray:
    """Query string -> flat trn_qnode array (see include/trinity_b200.h).  Mirrors the reference's operator subset and
    precedence (queries.cpp:11-27,477-520) followed by build_iterator's flattening (exec.cpp:328-400).
    `[a, b, c]` is a MatchSome group; like the reference's parser it starts with min = 1 and the application raises it:
    min_match sets match_some.min of every such group."""
    L = lib()
    nodes = np.zeros(256, dtype=QNODE_DTYPE)
    nn, root = C.c_uint32(), C.c_uint32()
    err = C.create_string_buffer(256)
    rc = L.trn_parse_query_dict(text.encode(), tdict._h, _ptr(nodes), len(nodes), C.byref(nn), C.byref(root), err, 256)
    if rc != 0:
        raise TrinityError(f"parse error: {err.value.decode()}")
    assert root.value == 0
    out = nodes[: nn.value].copy()
    if min_match is not None:
        out["term"][out["kind"] == NODE_SOME] = min_match
    return out


def debug_positions(codec: int, index: np.ndarray, hits: np.ndarray, term, docids) -> list:
    """per listed document the positions the kernels' own cursor code (csrc/hitcursor.h, run on the host) reads for one term"""
    index = np.ascontiguousarray(index, dtype=np.uint8)
    hits = np.ascontiguousarray(hits if hits is not None else np.zeros(0, np.uint8), dtype=np.uint8)
    t = TrnTerm(int(term[0]), int(term[1]), int(term[2]))
    d = _u32(list(docids))
    counts = np.zeros(max(len(d), 1), np.uint32)
    cap = 1 << 16
    while True:
        pos = np.zeros(cap, np.uint32)
        total = C.c_uint64()
        err = C.create_string_buffer(256)
        rc = lib().trn_debug_positions(codec, _ptr(index), index.size, _ptr(hits) if hits.size else None, hits.size, C.byref(t), _ptr(d), len(d), _ptr(counts),
                                       _ptr(pos), cap, C.byref(total), err, 256)
        if rc == -6:
            cap = int(total.value)
            continue
        if rc != 0:
            raise TrinityError(err.value.decode("utf-8", "replace") or f"rc={rc}")
        out, at = [], 0
        for i in range(len(d)):
            out.append(pos[at: at + int(counts[i])].copy())
            at += int(counts[i])
        return out


def debug_compile(codec: int, index: np.ndarray, terms: np.ndarray, nodes: np.ndarray, scored):
    """(steps, root_slot, nslots): the bitmap-path step program of one plan, compiled on the host (no GPU needed).
    scored: False / True, 2 = the DocumentsOnly program in its flat-tree form, 3 = flat-tree form with the masked second decode pass"""
    from ._ffi import STEP_DTYPE
    index = np.ascontiguousarray(index, dtype=np.uint8)
    terms = np.ascontiguousarray(terms, dtype=TERM_DTYPE)
    nodes = np.ascontiguousarray(nodes, dtype=QNODE_DTYPE)
    steps = np.zeros(512, STEP_DTYPE)
    n, rs, ns = C.c_uint32(), C.c_uint32(), C.c_uint32()
    err = C.create_string_buffer(256)
    rc = lib().trn_debug_compile(codec, _ptr(index), index.size, _ptr(terms), len(terms), _ptr(nodes), len(nodes), 0, int(scored), _ptr(steps), len(steps),
                                 C.byref(n), C.byref(rs), C.byref(ns), err, 256)
    if rc != 0:
        raise TrinityError(err.value.decode("utf-8", "replace"))
    return steps[: n.value].copy(), int(rs.value), int(ns.value)


def query_truth_table(nodes: np.ndarray):
    """(terms, table, necessary): the boolean function of a plan over its distinct terms as the candidate-driven planner sees it;
    table[a] (a = bit set of present terms, bit j = terms[j]) is True where the query matches"""
    nodes = np.ascontiguousarray(nodes, dtype=QNODE_DTYPE)
    terms = (C.c_uint32 * 8)()
    table = (C.c_uint32 * 8)()
    n, nec = C.c_uint32(), C.c_uint32()
    rc = lib().trn_query_truth_table(_ptr(nodes), len(nodes), 0, terms, C.byref(n), table, C.byref(nec))
    if rc != 0:
        raise TrinityError("query has more than 8 distinct terms (or a malformed tree)")
    tb_ = np.array([(table[a >> 5] >> (a & 31)) & 1 for a in range(1 << n.value)], bool)
    return [int(terms[j]) for j in range(n.value)], tb_, int(nec.value)


def _pack_queries(queries: Sequence[np.ndarray]):
    arr = (TrnQuery * len(queries))()
    keep = []
    for i, q in enumerate(queries):
        q = np.ascontiguousarray(q, dtype=QNODE_DTYPE)
        keep.append(q)
        arr[i].nodes = q.ctypes.data
        arr[i].nnodes = len(q)
        arr[i].root = 0
    return arr, keep


def debug_plan(codec: int, index: np.ndarray, terms: np.ndarray, queries: Sequence[np.ndarray], mode: int, k: int = 100, max_docid: int = 0):
    """(routes, (nslots, tree_slots)): the path (ROUTE_*) every query of the batch would run and the docset slots of the step-program and
    flat-tree launches, planned on the host as a GpuIndexSource created with this environment would (no GPU needed)"""
    index = np.ascontiguousarray(index, dtype=np.uint8)
    terms = np.ascontiguousarray(terms, dtype=TERM_DTYPE)
    arr, keep = _pack_queries(queries)
    routes = np.zeros(max(len(queries), 1), np.uint8)
    slots = (C.c_uint32 * 2)()
    err = C.create_string_buffer(256)
    rc = lib().trn_debug_plan(codec, _ptr(index), index.size, _ptr(terms), len(terms), max_docid, C.cast(arr, C.c_void_p), len(queries), mode, k,
                              _ptr(routes), slots, err, 256)
    if rc != 0:
        raise TrinityError(err.value.decode("utf-8", "replace") or f"rc={rc}")
    return routes[: len(queries)].copy(), (int(slots[0]), int(slots[1]))


def bm25_idf(doc_freq: int, docs_cnt: int) -> float:
    return float(lib().trn_bm25_idf(doc_freq, docs_cnt))


def bm25_score(idf: float, freq: int) -> float:
    return float(lib().trn_bm25_score(idf, freq))


# ----------------------------------------------------------------------------------------------- engine
@dataclass
class BatchResult:
    nq: int
    mode: int
    k: int
    offsets: np.ndarray       # nq+1
    docids: np.ndarray
    scores: Optional[np.ndarray]
    match_counts: np.ndarray  # nq
    postings_scanned: int
    index_bytes_touched: int
    kernel_launches: int
    device_ms: float
    exec_kernel_ms: float = 0.0
    # MODE_DOCS_COMPACT: what travelled from the device (the decoded docIDs above are produced on the host by trn_result_decode)
    total_words: int = 0
    nitems: int = 0
    raw: object = None  # copy=False: the TrnResult (ctx-owned buffers, valid until the next exec call); docids is None until decoded

    def result_bytes(self) -> int:
        """bytes of the result as it left the device: docIDs (+ scores) or compact words + segment descriptors"""
        if self.mode == MODE_DOCS_COMPACT:
            return 4 * self.total_words + 4 * self.nitems
        return 4 * int(self.offsets[-1]) * (1 if self.scores is None else 2)

    def decode_query(self, q: int, buf: Optional[np.ndarray] = None) -> np.ndarray:
        """MODE_DOCS_COMPACT with copy=False: query q's docIDs through trn_result_decode (== the consider() replay)"""
        n = int(self.match_counts[q])
        out = buf if buf is not None and len(buf) >= n else np.empty(max(n, 1), np.uint32)
        got = C.c_uint64()
        rc = lib().trn_result_decode(C.byref(self.raw), q, _ptr(out), len(out), C.byref(got))
        if rc != 0 or int(got.value) != n:
            raise TrinityError(f"trn_result_decode: rc={rc}, {got.value} docIDs, match_counts says {n}")
        return out[:n]

    def checksums(self) -> np.ndarray:
        """per-query sum of the matched docIDs (uint64, wrap-around): the full-size parity probe of bench.py"""
        if self.docids is not None:
            off = np.asarray(self.offsets, np.int64)
            cs = np.concatenate([np.zeros(1, np.uint64), np.cumsum(np.asarray(self.docids[: off[-1]], np.uint64), dtype=np.uint64)])
            return cs[off[1:]] - cs[off[:-1]]
        buf = np.empty(max(1, int(np.max(self.match_counts)) if self.nq else 1), np.uint32)
        return np.array([int(self.decode_query(q, buf).sum(dtype=np.uint64)) for q in range(self.nq)], np.uint64)

    def query(self, q: int):
        """(docids, scores) of query q.  top-k mode: only the valid entries, (score desc, docID asc)."""
        if self.docids is None:
            return self.decode_query(q).copy(), None
        a, b = int(self.offsets[q]), int(self.offsets[q + 1])
        d = self.docids[a:b]
        s = None if self.scores is None else self.scores[a:b]
        if self.mode == MODE_SCORED_TOPK:
            keep = s >= 0
            return d[keep], s[keep]
        return d, s


class GpuIndexSource:
    """== one device-resident IndexSource + AccessProxy (index_source.h:18-155, codecs.h:290-317) and the batch form of
    exec_query() (exec.h:50-52) over it."""

    def __init__(self, device: int = 0):
        self._L = lib()
        h = C.c_void_p()
        rc = self._L.trn_create(device, C.byref(h))
        self._h = h
        if rc != 0:
            msg = self._L.trn_last_error(h).decode() if h else "trn_create failed"
            raise TrinityError(msg)
        self.terms: Optional[np.ndarray] = None
        self.docs_cnt = 0

    def _ck(self, rc):
        if rc != 0:
            raise TrinityError(f"rc={rc}: " + self._L.trn_last_error(self._h).decode())

    def set_stream(self, cuda_stream_ptr: int):
        self._ck(self._L.trn_set_stream(self._h, C.c_void_p(cuda_stream_ptr)))

    def upload(self, codec: int, index: np.ndarray, terms: np.ndarray, max_docid: int):
        index = np.ascontiguousarray(index, dtype=np.uint8)
        terms = np.ascontiguousarray(terms, dtype=TERM_DTYPE)
        self._ck(self._L.trn_upload_index(self._h, codec, _ptr(index), index.size, _ptr(terms), len(terms), max_docid))
        self.terms = terms.copy()
        self.docs_cnt = max_docid
        self.codec = codec

    def upload_hits(self, index: np.ndarray, hits: np.ndarray):
        """LUCENE: hits.data of the uploaded index (== Lucene AccessProxy::hitsDataPtr) — needed for phrase plans"""
        index = np.ascontiguousarray(index, dtype=np.uint8)
        hits = np.ascontiguousarray(hits, dtype=np.uint8)
        self._ck(self._L.trn_upload_hits(self._h, _ptr(index), index.size, _ptr(hits) if hits.size else None, hits.size))

    def set_masked_documents(self, docids=None):
        """== masked_documents_registry: these docIDs never reach consider() / the top-k (None or empty clears)"""
        d = _u32([] if docids is None else docids)
        self._ck(self._L.trn_set_masked_documents(self._h, _ptr(d) if len(d) else None, len(d)))

    def info(self) -> dict:
        i = TrnIndexInfo()
        self._ck(self._L.trn_index_info_get(self._h, C.byref(i)))
        return {f: getattr(i, f) for f, _ in TrnIndexInfo._fields_}

    def set_bm25_weights(self, nodes: np.ndarray, docs_cnt: Optional[int] = None) -> np.ndarray:
        """fills TERM weights with ScorerWeight::idf (similarity.h:190-222) from the uploaded terms' document counts"""
        n = docs_cnt or self.docs_cnt
        for x in nodes:
            if x["kind"] == NODE_TERM and x["term"] != EMPTY_TERM:
                x["weight"] = bm25_idf(int(self.terms["documents"][x["term"]]), n)
        return nodes

    def _pack(self, queries: Sequence[np.ndarray]):
        return _pack_queries(queries)

    def exec_batch_device(self, queries: Sequence[np.ndarray], mode: int, k: int = 100, packed=None):
        arr, keep = packed if packed is not None else self._pack(queries)
        r = TrnResult()
        self._ck(self._L.trn_exec_batch_device(self._h, C.cast(arr, C.c_void_p), len(queries), mode, k, C.byref(r)))
        self._last = (mode, k, len(queries))
        return r

    def fetch(self) -> BatchResult:
        r = TrnResult()
        self._ck(self._L.trn_fetch_results(self._h, C.byref(r)))
        mode, k, nq = self._last
        return self._wrap(r, mode, k)

    def _wrap(self, r: TrnResult, mode: int, k: int, copy: bool = True) -> BatchResult:
        """copy=False returns views of the ctx-owned pinned host buffers (valid until the next exec call)"""
        nq = r.nq
        keep = (lambda a: a.copy()) if copy else (lambda a: a)
        offsets = keep(np.ctypeslib.as_array(r.offsets, shape=(nq + 1,)))
        n = int(offsets[nq])
        if mode == MODE_DOCS_COMPACT:
            counts = keep(np.ctypeslib.as_array(r.match_counts, shape=(nq,)))
            nitems = 0
            if nq and r.qitems:
                qi = np.ctypeslib.as_array(C.cast(r.qitems, C.POINTER(C.c_uint32)), shape=(nq, 4))
                nitems = int((qi[:, 0] + qi[:, 1]).max())
            br = BatchResult(nq, mode, k, offsets, None, None, counts, int(r.postings_scanned), int(r.index_bytes_touched), int(r.kernel_launches),
                             float(r.device_ms), float(r.exec_kernel_ms), total_words=int(r.total_words), nitems=nitems, raw=r)
            if copy:  # decode now: the ctx-owned buffers may be reused by the next call
                per = [br.decode_query(q).copy() for q in range(nq)]
                br.docids = np.concatenate(per) if per else np.zeros(0, np.uint32)
                br.offsets = np.concatenate([[0], np.cumsum([len(x) for x in per])]).astype(np.uint64)
                br.raw = None
            return br
        docids = keep(np.ctypeslib.as_array(r.docids, shape=(max(n, 1),))[:n])
        scores = None
        if mode != MODE_DOCS_ONLY:
            scores = keep(np.ctypeslib.as_array(r.scores, shape=(max(n, 1),))[:n])
        counts = keep(np.ctypeslib.as_array(r.match_counts, shape=(nq,)))
        return BatchResult(nq, mode, k, offsets, docids, scores, counts, int(r.postings_scanned), int(r.index_bytes_touched),
                           int(r.kernel_launches), float(r.device_ms), float(r.exec_kernel_ms))

    def pack(self, queries: Sequence[np.ndarray]):
        """pre-marshal a batch of plans (trn_query array); pass the result to exec_batch(..., packed=...) to keep ctypes
        marshalling out of a timed region"""
        return self._pack(queries)

    def exec_batch(self, queries: Sequence[np.ndarray], mode: int, k: int = 100, copy: bool = True, packed=None) -> BatchResult:
        """== exec_query() for a batch: plans H2D, fused kernels, results D2H."""
        arr, keep = packed if packed is not None else self._pack(queries)
        r = TrnResult()
        self._ck(self._L.trn_exec_batch(self._h, C.cast(arr, C.c_void_p), len(queries), mode, k, C.byref(r)))
        self._last = (mode, k, len(queries))
        return self._wrap(r, mode, k, copy)

    def last_timings(self) -> dict:
        """host-side breakdown (ms) of the last exec_batch / exec_batch_device call"""
        t = TrnTimings()
        self._ck(self._L.trn_last_timings(self._h, C.byref(t)))
        return {n: float(getattr(t, n)) for n, _ in TrnTimings._fields_}

    def last_routes(self) -> np.ndarray:
        """debug: the path (ROUTE_*) every query of the last exec_batch / exec_batch_device call ran"""
        n = C.c_uint32()
        out = np.zeros(max(getattr(self, "_last", (0, 0, 0))[2], 1), np.uint8)
        self._ck(self._L.trn_debug_last_routes(self._h, _ptr(out), len(out), C.byref(n)))
        return out[: n.value].copy()

    def last_topk_device(self):
        d, s, c = C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._ck(self._L.trn_last_topk_device(self._h, C.byref(d), C.byref(s), C.byref(c)))
        return d.value, s.value, c.value

    def merge_topk(self, docids_ptr: int, scores_ptr: int, nshards: int, nq: int, k: int, out_docids_ptr: int, out_scores_ptr: int):
        self._ck(self._L.trn_merge_topk(self._h, C.c_void_p(docids_ptr), C.c_void_p(scores_ptr), nshards, nq, k,
                                        C.c_void_p(out_docids_ptr), C.c_void_p(out_scores_ptr)))

    def decode_terms(self, term_ids: Iterable[int], materialise: bool = True):
        """== PostingsListIterator::next() over whole lists.  Returns (docids, freqs, sums[nterms,2], device_ms)."""
        t = _u32(list(term_ids))
        total = int(self.terms["documents"][t].sum())
        d = np.zeros(total if materialise else 0, np.uint32)
        f = np.zeros(total if materialise else 0, np.uint32)
        sums = np.zeros((len(t), 2), np.uint64)
        ms = C.c_float()
        self._ck(self._L.trn_decode_terms(self._h, _ptr(t), len(t), int(materialise), _ptr(d) if materialise else None,
                                          _ptr(f) if materialise else None, _ptr(sums), C.byref(ms)))
        return d, f, sums, float(ms.value)

    def encode_google(self, lists, block_docs: int = 32, skiplist_step: int = 8, countdown: Optional[int] = None):
        """GPU-side Encoder (== Codecs::Google::Encoder, google_codec.cpp:9-176): builds the GOOGLE index of `lists` on the device.
        lists: one (docids, freqs[, positions]) per term — positions (all of them or none) = the hits of the term's postings, concatenated.
        Returns (index bytes, terms array, countdown after the last term, device_ms)."""
        lists = list(lists)
        with_pos = len(lists) > 0 and len(lists[0]) > 2 and lists[0][2] is not None
        tb = np.zeros(len(lists) + 1, np.uint64)
        for i, l in enumerate(lists):
            tb[i + 1] = tb[i] + len(l[0])
        d = np.concatenate([_u32(l[0]) for l in lists]) if lists else np.zeros(0, np.uint32)
        f = np.concatenate([_u32(l[1]) for l in lists]) if lists else np.zeros(0, np.uint32)
        p = np.concatenate([_u32(l[2]) for l in lists]) if with_pos else None
        terms = np.zeros(len(lists), dtype=TERM_DTYPE)
        cd = C.c_uint32(countdown if countdown is not None else skiplist_step)
        nbytes, ms = C.c_uint64(), C.c_float()
        cap = 16 + 2 * len(lists) + int(d.size) * 11 + (int(f.sum()) * 5 if with_pos else int(f.sum())) + 8 * (int(d.size) // max(1, block_docs) + len(lists) + 1)
        out = np.zeros(cap, np.uint8)
        self._ck(self._L.trn_encode_google(self._h, _ptr(tb), len(lists), _ptr(d), _ptr(f), _ptr(p), block_docs, skiplist_step, C.byref(cd),
                                           _ptr(out), cap, C.byref(nbytes), _ptr(terms), C.byref(ms)))
        return out[:nbytes.value].copy(), terms, int(cd.value), float(ms.value)

    def close(self):
        if getattr(self, "_h", None):
            self._L.trn_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def directory_probe(codec: int, index: np.ndarray, term: tuple):
    """Host-side block directory of one term: (blk_last[nblocks+1], blk_off[nblocks+1], first_doc)."""
    L = lib()
    index = np.ascontiguousarray(index, dtype=np.uint8)
    t = TrnTerm(int(term[0]), int(term[1]), int(term[2]))
    nb, fd = C.c_uint32(), C.c_uint32()
    err = C.create_string_buffer(256)
    cap = int(term[0]) + 4  # (block sizes below 32 exist in sweep indexes)
    last, off = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
    rc = L.trn_directory_probe(codec, _ptr(index), index.size, C.byref(t), _ptr(last), _ptr(off), cap, C.byref(nb), C.byref(fd), err, 256)
    if rc != 0:
        raise TrinityError(err.value.decode())
    n = nb.value + (1 if nb.value else 0)
    return last[:n], off[:n], fd.value


def directory_lookup(codec: int, index: np.ndarray, term: tuple, docids):
    """(blocks, tf_shift, tf_entries): first block of the term whose last docID >= docids[i], through the kernels' own lookup code on the host"""
    index = np.ascontiguousarray(index, dtype=np.uint8)
    t = TrnTerm(int(term[0]), int(term[1]), int(term[2]))
    d = _u32(docids)
    out = np.zeros(len(d), np.uint32)
    sh, ne = C.c_uint32(), C.c_uint32()
    err = C.create_string_buffer(256)
    rc = lib().trn_directory_lookup(codec, _ptr(index), index.size, C.byref(t), _ptr(d), len(d), _ptr(out), C.byref(sh), C.byref(ne), err, 256)
    if rc != 0:
        raise TrinityError(err.value.decode("utf-8", "replace"))
    return out, int(sh.value), int(ne.value)


def directory_stats(codec: int, index: np.ndarray, terms: np.ndarray, threads: int = 1) -> dict:
    """size of the load-time directory trn_upload_index would build for this index (host only)"""
    index = np.ascontiguousarray(index, dtype=np.uint8)
    terms = np.ascontiguousarray(terms, dtype=TERM_DTYPE)
    db, nb, te = C.c_uint64(), C.c_uint64(), C.c_uint64()
    err = C.create_string_buffer(256)
    rc = lib().trn_directory_stats(codec, _ptr(index), index.size, _ptr(terms), len(terms), threads, C.byref(db), C.byref(nb), C.byref(te), err, 256)
    if rc != 0:
        raise TrinityError(err.value.decode("utf-8", "replace"))
    return {"directory_bytes": db.value, "total_blocks": nb.value, "table_entries": te.value, "index_bytes": int(index.size)}


class Segment:
    """A segment directory written by Trinity's SegmentIndexSession::commit() (indexer.cpp:241-300) — the host half of
    SegmentIndexSource (segment_index_source.cpp:5-186)."""

    def __init__(self, path: str):
        self._L = lib()
        h = C.c_void_p()
        err = C.create_string_buffer(512)
        if self._L.trn_segment_open(str(path).encode(), C.byref(h), err, 512) != 0:
            raise TrinityError(f"segment {path}: {err.value.decode('utf-8', 'replace')}")
        self._h = h
        codec, nt, nm = C.c_int(), C.c_uint32(), C.c_uint64()
        ib, sth, std_ = C.c_uint64(), C.c_uint64(), C.c_uint64()
        tt, dc = C.c_uint32(), C.c_uint32()
        self._L.trn_segment_info(h, C.byref(codec), C.byref(nt), C.byref(ib), C.byref(sth), C.byref(tt), C.byref(std_), C.byref(dc), C.byref(nm))
        self.codec = codec.value
        self.field_statistics = {"sumTermHits": sth.value, "totalTerms": tt.value, "sumTermsDocs": std_.value, "docsCnt": dc.value}
        p, n = C.c_void_p(), C.c_uint64()
        self._L.trn_segment_index(h, C.byref(p), C.byref(n))
        self.index = (np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n.value,)) if n.value else np.zeros(0, np.uint8))
        tp, npp, tn = C.c_void_p(), C.c_void_p(), C.c_uint32()
        self._L.trn_segment_terms(h, C.byref(tp), C.byref(npp), C.byref(tn))
        if tn.value:
            self.terms = np.ctypeslib.as_array(C.cast(tp, C.POINTER(C.c_uint8)), shape=(tn.value * 12,)).view(TERM_DTYPE).copy()
            arr = C.cast(npp, C.POINTER(C.c_char_p))
            self.names = [arr[i].decode("utf-8", "surrogateescape") for i in range(tn.value)]  # term names are bytes (str8_t)
        else:
            self.terms, self.names = np.zeros(0, TERM_DTYPE), []
        mp, mn = C.c_void_p(), C.c_uint64()
        self._L.trn_segment_masked(h, C.byref(mp), C.byref(mn))
        self.masked_documents = (np.ctypeslib.as_array(C.cast(mp, C.POINTER(C.c_uint32)), shape=(mn.value,)).copy() if mn.value
                                 else np.zeros(0, np.uint32))

    def upload(self, gpu: "GpuIndexSource", max_docid: int):
        gpu.upload(self.codec, self.index, self.terms, max_docid)
        return TermDictionary(self.names)

    def __del__(self):
        try:
            self._L.trn_segment_close(self._h)
        except Exception:
            pass
