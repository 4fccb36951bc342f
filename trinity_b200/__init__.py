"""trinity_b200 — GPU-native (H100, sm_90a) execution engine for Trinity's inverted-index hot path.

Thin Python plumbing over the C ABI (include/trinity_b200.h).  Class and method names follow the reference's
domain vocabulary (IndexSession/Encoder, IndexSource, exec_query, term_index_ctx, postings, docsets);
all decode / docset / scoring work happens in the sm_90a kernels of libtrinity_b200.so — there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Iterable, List, Optional, Sequence

import numpy as np

from ._ffi import (HIT_DTYPE, QNODE_DTYPE, TERM_DTYPE, TrnIndexInfo, TrnIntersections, TrnIsectReq, TrnMatches, TrnPercolation, TrnPercolatorInfo, TrnQuery,
                   TrnIndexed, TrnMerged, TrnMergeSource, TrnResult, TrnTerm, TrnTimings, lib)

CODEC_GOOGLE, CODEC_LUCENE = 0, 1
MODE_DOCS_ONLY, MODE_SCORED_ALL, MODE_SCORED_TOPK = 0, 1, 2  # == ExecFlags::DocumentsOnly / AccumulatedScoreScheme (+ fused top-k sink)
MODE_MATCHED_TERMS = 4  # no ExecFlags: every match with the query terms it holds and their hits (GpuIndexSource.exec_matches)
MODE_DOCS_COMPACT = 3  # DocumentsOnly, compact result segments (bitmap / bucketed 8-bit offsets / 16-bit offsets / docIDs per tile): trn_result_decode replays them
NODE_TERM, NODE_AND, NODE_OR, NODE_NOT, NODE_OPTIONAL, NODE_SOME, NODE_PHRASE = 0, 1, 2, 3, 4, 5, 6
# the path a query ran (GpuIndexSource.last_routes, == TRN_ROUTE_* of include/trinity_b200.h)
ROUTE_STEPS, ROUTE_FLAT_AND, ROUTE_FLAT_OR, ROUTE_CANDIDATE, ROUTE_SCORE_FLAT, ROUTE_FLAT_TREE, ROUTE_EXEC_TILES = 0, 1, 2, 3, 4, 5, 6
EMPTY_TERM = 0xFFFFFFFF
DENSE_NONE = 0xFFFFFFFF  # debug_dense_terms: the term has no resident bitmap
DOC_IDS_END = 0xFFFFFFFF  # DocIDsEND, common.h:43
DOCSET_NONE = 0xFFFFFFFF  # trn_doc_filter: no allow / deny set


class TrinityError(RuntimeError):
    pass


def _u32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.uint32)


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _payload_arrays(lists):
    """the per-hit payload sizes (uint8) and payloads (uint64) of (docids, freqs, positions, payload_lens, payloads) terms, concatenated"""
    pl = np.ascontiguousarray(np.concatenate([np.asarray(l[3], np.uint8) for l in lists]), np.uint8)
    pv = np.ascontiguousarray(np.concatenate([np.asarray(l[4], np.uint64) for l in lists]), np.uint64)
    if len(pl) != len(pv):
        raise TrinityError("one payload length and one payload per hit")
    return pl, pv


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

    def term_id(self, name: str) -> int:
        """the term's id, EMPTY_TERM when the dictionary does not hold it"""
        if not hasattr(self, "_ids"):
            self._ids = {n: i for i, n in enumerate(self.names)}
        return self._ids.get(name, EMPTY_TERM)

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
    scored: False / True, 2 = the DocumentsOnly program in its flat-tree form"""
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


def debug_dense_runs(codec: int, index: np.ndarray, terms: np.ndarray, queries: Sequence[np.ndarray], mode: int, k: int = 100, max_docid: int = 0):
    """(qtiles, tickets): the same plan's (tile_lo, ntiles) of every query, and the run-major tickets of its all-bitmap flat ANDs in launch
    order, one row (query, first tile, end tile) each — the tiles [first, end) of one 2^17-docID run"""
    return _debug_run_tickets(lib().trn_debug_dense_runs, codec, index, terms, queries, mode, k, max_docid)


def debug_mixed_runs(codec: int, index: np.ndarray, terms: np.ndarray, queries: Sequence[np.ndarray], mode: int, k: int = 100, max_docid: int = 0):
    """as debug_dense_runs, for the flat ANDs with exactly one operand without a resident bitmap"""
    return _debug_run_tickets(lib().trn_debug_mixed_runs, codec, index, terms, queries, mode, k, max_docid)


def debug_cand_runs(codec: int, index: np.ndarray, terms: np.ndarray, queries: Sequence[np.ndarray], mode: int, k: int = 100, max_docid: int = 0):
    """(qgroups, tickets): the candidate-driven queries' run-major tickets as the planner lays them out (no GPU needed).  qgroups[q, 1] is
    query q's count of 32-block lead groups; a ticket row is (query, group, the group's first docID), ordered by that docID's 2^17-docID run,
    queries ascending within a run.  Empty with TRN_CAND_RUNS=0, on LUCENE, in the scored modes and beside a phrase plan."""
    return _debug_run_tickets(lib().trn_debug_cand_runs, codec, index, terms, queries, mode, k, max_docid)


def _debug_run_tickets(fn, codec, index, terms, queries, mode, k, max_docid):
    index = np.ascontiguousarray(index, dtype=np.uint8)
    terms = np.ascontiguousarray(terms, dtype=TERM_DTYPE)
    arr, keep = _pack_queries(queries)
    qtiles = np.zeros((max(len(queries), 1), 2), np.uint32)
    n = C.c_uint64()
    err = C.create_string_buffer(256)
    args = (codec, _ptr(index), index.size, _ptr(terms), len(terms), max_docid, C.cast(arr, C.c_void_p), len(queries), mode, k, _ptr(qtiles))
    rc = fn(*args, None, 0, C.byref(n), err, 256)
    tickets = np.zeros((max(n.value, 1), 3), np.uint32)
    if rc == -6:  # TRN_ERR_CAPACITY: sized, now filled
        rc = fn(*args, _ptr(tickets), n.value, C.byref(n), err, 256)
    if rc != 0:
        raise TrinityError(err.value.decode("utf-8", "replace") or f"rc={rc}")
    return qtiles[: len(queries)].copy(), tickets[: n.value].copy()


def debug_dense_terms(codec: int, index: np.ndarray, terms: np.ndarray):
    """(offsets, bitmap_bytes): the first 32-bit word of every term's resident docID bitmap (DENSE_NONE: none) and the bytes of all of them,
    selected on the host as a GpuIndexSource created with this environment would on upload (no GPU needed)"""
    off, n, nbytes = _debug_bitmap_terms(lib().trn_debug_dense_terms, codec, index, terms)
    assert int(np.count_nonzero(off != DENSE_NONE)) == n
    return off, nbytes


def debug_probe_terms(codec: int, index: np.ndarray, terms: np.ndarray):
    """(offsets, nselected, bitmap_bytes) of the probe bitmaps, the second tier that candidate-driven conjunctions probe: per term the word
    its probes read from (its dense bitmap's, its probe bitmap's, DENSE_NONE: neither), the number of probe-tier terms and their bytes,
    selected on the host as a GpuIndexSource created with this environment would on upload (no GPU needed)"""
    return _debug_bitmap_terms(lib().trn_debug_probe_terms, codec, index, terms)


def _debug_bitmap_terms(fn, codec, index, terms):
    index = np.ascontiguousarray(index, dtype=np.uint8)
    terms = np.ascontiguousarray(terms, dtype=TERM_DTYPE)
    off = np.zeros(max(len(terms), 1), np.uint32)
    n, nbytes = C.c_uint32(), C.c_uint64()
    err = C.create_string_buffer(256)
    rc = fn(codec, _ptr(index), index.size, _ptr(terms), len(terms), _ptr(off), C.byref(n), C.byref(nbytes), err, 256)
    if rc != 0:
        raise TrinityError(err.value.decode("utf-8", "replace") or f"rc={rc}")
    return off[: len(terms)].copy(), n.value, int(nbytes.value)


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


def debug_hits(codec: int, index: np.ndarray, hits: np.ndarray, term, docids) -> list:
    """per listed document None when the term does not hold it, else (freq, positions, payload_lens, payloads) as the kernels' hit walker
    (csrc/hitcursor.h HitWalker, run on the host) reads them for one term"""
    index = np.ascontiguousarray(index, dtype=np.uint8)
    hits = np.ascontiguousarray(hits if hits is not None else np.zeros(0, np.uint8), dtype=np.uint8)
    t = TrnTerm(int(term[0]), int(term[1]), int(term[2]))
    d = _u32(list(docids))
    counts = np.zeros(max(len(d), 1), np.uint32)
    found = np.zeros(max(len(d), 1), np.uint8)
    cap = 1 << 16
    while True:
        out = np.zeros(cap, HIT_DTYPE)
        total = C.c_uint64()
        err = C.create_string_buffer(256)
        rc = lib().trn_debug_hits(codec, _ptr(index), index.size, _ptr(hits) if hits.size else None, hits.size, C.byref(t), _ptr(d), len(d), _ptr(found),
                                  _ptr(counts), out.ctypes.data, cap, C.byref(total), err, 256)
        if rc == -6:
            cap = int(total.value)
            continue
        if rc != 0:
            raise TrinityError(err.value.decode("utf-8", "replace") or f"rc={rc}")
        res, at = [], 0
        for i in range(len(d)):
            if not found[i]:
                res.append(None)
                continue
            h = out[at: at + int(counts[i])]
            res.append((int(counts[i]), h["pos"].copy(), h["payload_len"].copy(), h["payload"].copy()))
            at += int(counts[i])
        return res


class MatchesResult:
    """trn_exec_matches: per query its matches (ascending docID), per match its terms (ascending term index) and freqs, per term its
    hits (HIT_DTYPE: payload, pos, payload_len)"""

    def __init__(self, r: TrnMatches):
        nq, nm, nt, nh = int(r.nq), int(r.total_matches), int(r.total_terms), int(r.total_hits)
        self.nq = nq
        self.doc_offsets = np.ctypeslib.as_array(r.doc_offsets, shape=(nq + 1,)).copy()
        self.docids = np.ctypeslib.as_array(r.docids, shape=(max(nm, 1),))[:nm].copy()
        self.term_offsets = np.ctypeslib.as_array(r.term_offsets, shape=(nm + 1,)).copy()
        self.terms = np.ctypeslib.as_array(r.terms, shape=(max(nt, 1),))[:nt].copy()
        self.freqs = np.ctypeslib.as_array(r.freqs, shape=(max(nt, 1),))[:nt].copy()
        self.hit_offsets = np.ctypeslib.as_array(r.hit_offsets, shape=(nt + 1,)).copy()
        raw = (C.c_uint8 * (max(nh, 1) * HIT_DTYPE.itemsize)).from_address(r.hits)
        self.hits = np.frombuffer(raw, dtype=HIT_DTYPE, count=max(nh, 1))[:nh].copy()
        self.device_ms, self.docs_ms, self.chunks = float(r.device_ms), float(r.docs_ms), int(r.chunks)
        self.count_ms, self.write_ms = float(r.count_ms), float(r.write_ms)

    def query(self, q: int) -> np.ndarray:
        return self.docids[int(self.doc_offsets[q]): int(self.doc_offsets[q + 1])]

    def matches(self, q: int):
        """== the consider(const matched_document &) stream of query q: (docid, [(term, freq, positions, payload_lens, payloads)])"""
        for m in range(int(self.doc_offsets[q]), int(self.doc_offsets[q + 1])):
            terms = []
            for t in range(int(self.term_offsets[m]), int(self.term_offsets[m + 1])):
                h = self.hits[int(self.hit_offsets[t]): int(self.hit_offsets[t + 1])]
                terms.append((int(self.terms[t]), int(self.freqs[t]), h["pos"], h["payload_len"], h["payload"]))
            yield int(self.docids[m]), terms


def debug_intersect_plan(masks, firsts, max_masks: int = 0):
    """the host step of GpuIndexSource.intersect (csrc/isectplan.h) on one request's distinct masks and their first docIDs ->
    (epoch_start, [epoch arrays as [(mask, final index or -1)]], final antichain)"""
    m = np.ascontiguousarray(masks, np.uint64)
    f = _u32(firsts)
    n = len(m)
    es, eo, fm = np.zeros(max(n, 1), np.uint32), np.zeros(n + 1, np.uint32), np.zeros(max(n, 1), np.uint64)
    ne, nent, nf = C.c_uint32(), C.c_uint64(), C.c_uint32()
    err = C.create_string_buffer(256)
    cap = 1 << 12
    while True:
        sm, ss = np.zeros(cap, np.uint64), np.zeros(cap, np.int32)
        rc = lib().trn_debug_intersect_plan(_ptr(m), _ptr(f), n, max_masks, _ptr(es), _ptr(eo), _ptr(sm), _ptr(ss), cap, C.byref(ne), C.byref(nent),
                                            _ptr(fm), C.byref(nf), err, 256)
        if rc == -6 and nent.value > cap:
            cap = nent.value
            continue
        if rc != 0:
            raise TrinityError(f"rc={rc}: {err.value.decode()}")
        break
    arrays = [[(int(sm[i]), int(ss[i])) for i in range(int(eo[e]), int(eo[e + 1]))] for e in range(ne.value)]
    return [int(x) for x in es[: ne.value]], arrays, [int(x) for x in fm[: nf.value]]


class IntersectResult:
    """GpuIndexSource.intersect_batch: per request its [(mask, count)] in finalize()'s order (popcount, then count, descending; ties by mask),
    and the device times of the two passes and the host time of the planner between them"""

    def __init__(self, r: TrnIntersections):
        n, tot = int(r.n), int(r.total)
        offs = np.ctypeslib.as_array(r.offsets, shape=(n + 1,)).copy() if n else np.zeros(1, np.uint64)
        masks = np.ctypeslib.as_array(r.masks, shape=(max(tot, 1),))[:tot].copy() if tot else np.zeros(0, np.uint64)
        counts = np.ctypeslib.as_array(r.counts, shape=(max(tot, 1),))[:tot].copy() if tot else np.zeros(0, np.uint32)
        self.results = [[(int(masks[j]), int(counts[j])) for j in range(int(offs[i]), int(offs[i + 1]))] for i in range(n)]
        self.postings, self.distinct = int(r.postings), int(r.distinct)
        self.masks_ms, self.plan_ms, self.count_ms, self.total_ms = float(r.masks_ms), float(r.plan_ms), float(r.count_ms), float(r.total_ms)

    def __getitem__(self, i: int):
        return self.results[i]

    def __len__(self):
        return len(self.results)


class DocSet:
    """A resident docID set of one GpuIndexSource (trn_docset_create): the allow or deny side of a query's document filter.  It lives
    until close() or the source's next upload; any number of queries and batches may use it."""

    def __init__(self, source: "GpuIndexSource", handle: int, size: int):
        self.source, self.handle, self.size = source, handle, size

    def close(self):
        if self.handle is not None and self.source._h:
            self.source._ck(self.source._L.trn_docset_destroy(self.source._h, self.handle))
        self.handle = None


@dataclass(frozen=True)
class DocFilter:
    """== an IndexDocumentsFilter over docID sets: a query ignores d iff (allow and d not in allow) or (deny and d in deny), beside the
    masked documents"""
    allow: Optional[DocSet] = None
    deny: Optional[DocSet] = None


def _pack_filters(filters: Optional[Sequence[Optional[DocFilter]]], nq: int, source=None) -> Optional[np.ndarray]:
    """one trn_doc_filter (allow, deny handles) per query; None -> None (the call without filters)"""
    if filters is None:
        return None
    if len(filters) != nq:
        raise ValueError(f"{len(filters)} filters for {nq} queries")
    out = np.full((nq, 2), DOCSET_NONE, np.uint32)
    for q, f in enumerate(filters):
        if f is None:
            continue
        for j, d in enumerate((f.allow, f.deny)):
            if d is None:
                continue
            if d.handle is None:
                raise ValueError(f"query {q}: a closed DocSet")
            if source is not None and d.source is not source:
                raise ValueError(f"query {q}: a DocSet of another index source")
            out[q, j] = d.handle
    return out


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

    def docset(self, docids) -> DocSet:
        """a resident docID set for DocFilter (trn_docset_create): order and duplicates do not matter, docIDs above max_docid are
        ignored, docID 0 is refused; an empty set is valid (as an allow set it matches nothing)"""
        d = _u32(docids)
        h = C.c_uint32()
        self._ck(self._L.trn_docset_create(self._h, _ptr(d) if len(d) else None, len(d), C.byref(h)))
        return DocSet(self, int(h.value), len(d))

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

    def exec_batch_device(self, queries: Sequence[np.ndarray], mode: int, k: int = 100, packed=None, filters=None):
        """filters: None, or one None / DocFilter per query"""
        arr, keep = packed if packed is not None else self._pack(queries)
        r = TrnResult()
        f = _pack_filters(filters, len(queries), self)
        if f is None:
            self._ck(self._L.trn_exec_batch_device(self._h, C.cast(arr, C.c_void_p), len(queries), mode, k, C.byref(r)))
        else:
            self._ck(self._L.trn_exec_batch_device_filtered(self._h, C.cast(arr, C.c_void_p), len(queries), mode, k, _ptr(f), C.byref(r)))
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

    def exec_batch(self, queries: Sequence[np.ndarray], mode: int, k: int = 100, copy: bool = True, packed=None, filters=None) -> BatchResult:
        """== exec_query() for a batch: plans H2D, fused kernels, results D2H.  filters: None, or one None / DocFilter per query (the
        IndexDocumentsFilter of exec_query)"""
        arr, keep = packed if packed is not None else self._pack(queries)
        r = TrnResult()
        f = _pack_filters(filters, len(queries), self)
        if f is None:
            self._ck(self._L.trn_exec_batch(self._h, C.cast(arr, C.c_void_p), len(queries), mode, k, C.byref(r)))
        else:
            self._ck(self._L.trn_exec_batch_filtered(self._h, C.cast(arr, C.c_void_p), len(queries), mode, k, _ptr(f), C.byref(r)))
        self._last = (mode, k, len(queries))
        return self._wrap(r, mode, k, copy)

    def exec_matches(self, queries: Sequence[np.ndarray], packed=None, filters=None) -> MatchesResult:
        """== exec_query() with no ExecFlags for a batch: every match with the query terms it holds and their hits (TRN_MODE_MATCHED_TERMS).
        filters: None, or one None / DocFilter per query"""
        arr, keep = packed if packed is not None else self._pack(queries)
        r = TrnMatches()
        f = _pack_filters(filters, len(queries), self)
        if f is None:
            self._ck(self._L.trn_exec_matches(self._h, C.cast(arr, C.c_void_p), len(queries), C.byref(r)))
        else:
            self._ck(self._L.trn_exec_matches_filtered(self._h, C.cast(arr, C.c_void_p), len(queries), _ptr(f), C.byref(r)))
        self._last = (MODE_MATCHED_TERMS, 0, len(queries))
        return MatchesResult(r)

    def intersect_batch(self, requests: Sequence[Sequence[Sequence[int]]], stopwords_mask: int = 0) -> IntersectResult:
        """== Trinity::intersect_impl(stopwordsMask, tokens, src, maskedDocumentsRegistry) (intersect.cpp:5-170) for every request in one
        call: a request is a list of up to 64 groups of synonymous term ids (EMPTY_TERM: a token the source does not know); bit g of a
        result mask stands for group g.  The masked documents set on this source are the registry."""
        keep, arr = [], (TrnIsectReq * max(len(requests), 1))()
        for i, groups in enumerate(requests):
            offs = _u32(np.concatenate([[0], np.cumsum([len(g) for g in groups])]) if len(groups) else [0])
            terms = _u32([t for g in groups for t in g] or [0])
            keep += [offs, terms]
            arr[i] = TrnIsectReq(offs.ctypes.data, terms.ctypes.data, len(groups), stopwords_mask)
        r = TrnIntersections()
        self._ck(self._L.trn_intersect(self._h, C.cast(arr, C.c_void_p), len(requests), C.byref(r)))
        return IntersectResult(r)

    def intersect(self, groups: Sequence[Sequence[int]], stopwords_mask: int = 0):
        """one request of intersect_batch -> [(mask, count)]"""
        return self.intersect_batch([groups], stopwords_mask)[0]

    def intersect_tokens(self, token_groups: Sequence[Sequence[str]], tdict: "TermDictionary", stopwords_mask: int = 0):
        """intersect() with the tokens named: each resolved through the source's dictionary (unknown names are unknown tokens)"""
        return self.intersect([[tdict.term_id(t) for t in g] for g in token_groups], stopwords_mask)

    def last_timings(self) -> dict:
        """host-side breakdown (ms) of the last exec_batch / exec_batch_device call"""
        t = TrnTimings()
        self._ck(self._L.trn_last_timings(self._h, C.byref(t)))
        return {n: float(getattr(t, n)) for n, _ in TrnTimings._fields_}

    def dense_bitmap(self, term: int):
        """debug: (base docID, words) of the term's resident bitmap as the upload built it (bit b of word w = docID base + 32 w + b), or None"""
        base, n = C.c_uint64(), C.c_uint64()
        rc = self._L.trn_debug_dense_bitmap(self._h, term, None, 0, C.byref(base), C.byref(n))  # sizes it (TRN_ERR_CAPACITY when it exists)
        if n.value == 0:
            self._ck(rc)
            return None
        out = np.zeros(n.value, np.uint32)
        self._ck(self._L.trn_debug_dense_bitmap(self._h, term, _ptr(out), n.value, C.byref(base), C.byref(n)))
        return int(base.value), out

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
        lists: one (docids, freqs[, positions[, payload_lens, payloads]]) per term — positions (all of them or none) = the hits of the
        term's postings, concatenated; payload_lens (uint8, 0..8) / payloads (uint64, the payload in its low bytes) one per hit, all terms
        or none (trn_encode_google_payloads).  Returns (index bytes, terms array, countdown after the last term, device_ms)."""
        lists = list(lists)
        with_pos = len(lists) > 0 and len(lists[0]) > 2 and lists[0][2] is not None
        with_pay = with_pos and len(lists[0]) > 4 and lists[0][3] is not None
        tb = np.zeros(len(lists) + 1, np.uint64)
        for i, l in enumerate(lists):
            tb[i + 1] = tb[i] + len(l[0])
        d = np.concatenate([_u32(l[0]) for l in lists]) if lists else np.zeros(0, np.uint32)
        f = np.concatenate([_u32(l[1]) for l in lists]) if lists else np.zeros(0, np.uint32)
        p = np.concatenate([_u32(l[2]) for l in lists]) if with_pos else None
        pl, pv = _payload_arrays(lists) if with_pay else (None, None)
        terms = np.zeros(len(lists), dtype=TERM_DTYPE)
        cd = C.c_uint32(countdown if countdown is not None else skiplist_step)
        nbytes, ms = C.c_uint64(), C.c_float()
        cap = 16 + 2 * len(lists) + int(d.size) * 11 + (int(f.sum()) * 5 if with_pos else int(f.sum())) + 8 * (int(d.size) // max(1, block_docs) + len(lists) + 1)
        if with_pay:
            cap += 9 * int(f.sum())  # a size byte and up to 8 payload bytes per hit
        out = np.zeros(cap, np.uint8)
        self._ck(self._L.trn_encode_google_payloads(self._h, _ptr(tb), len(lists), _ptr(d), _ptr(f), _ptr(p), _ptr(pl), _ptr(pv), block_docs, skiplist_step,
                                                    C.byref(cd), _ptr(out), cap, C.byref(nbytes), _ptr(terms), C.byref(ms)))
        return out[:nbytes.value].copy(), terms, int(cd.value), float(ms.value)

    def encode_lucene(self, lists):
        """GPU-side Encoder (== Codecs::Lucene::Encoder, lucene_codec.cpp:163-388): builds the LUCENE index and its hits.data on the device.
        lists: one (docids, freqs[, positions[, payload_lens, payloads]]) per term, as for encode_google.  Returns (index bytes, hits bytes,
        terms array, device_ms)."""
        lists = list(lists)
        with_pos = len(lists) > 0 and len(lists[0]) > 2 and lists[0][2] is not None
        with_pay = with_pos and len(lists[0]) > 4 and lists[0][3] is not None
        pl, pv = _payload_arrays(lists) if with_pay else (None, None)
        tb = np.zeros(len(lists) + 1, np.uint64)
        for i, l in enumerate(lists):
            tb[i + 1] = tb[i] + len(l[0])
        d = np.concatenate([_u32(l[0]) for l in lists]) if lists else np.zeros(0, np.uint32)
        f = np.concatenate([_u32(l[1]) for l in lists]) if lists else np.zeros(0, np.uint32)
        p = np.concatenate([_u32(l[2]) for l in lists]) if with_pos else None
        terms = np.zeros(len(lists), dtype=TERM_DTYPE)
        nhits = int(f.sum(dtype=np.uint64))
        # upper bounds: an int-block is at most 1 + 4 * 166 bytes, so a full document block (two of them) < 11 bytes per document, a tail
        # document <= 10; a full hit block (int-block + 3) < 6 bytes per hit, a tail hit <= 3 (deltas < 2^14)
        icap = 16 + 14 * len(lists) + 11 * int(d.size) + 22 * (int(d.size) // 128)
        hcap = 16 + 6 * nhits + (9 * nhits if with_pay else 0)  # with payloads: up to a size byte (or its int-block) and 8 bytes per hit
        index, hits = np.empty(icap, np.uint8), np.empty(hcap, np.uint8)
        nb, hb, ms = C.c_uint64(), C.c_uint64(), C.c_float()
        self._ck(self._L.trn_encode_lucene_payloads(self._h, _ptr(tb), len(lists), _ptr(d), _ptr(f), _ptr(p), _ptr(pl), _ptr(pv), _ptr(index), icap,
                                                    C.byref(nb), _ptr(hits), hcap, C.byref(hb), _ptr(terms), C.byref(ms)))
        return index[:nb.value].copy(), hits[:hb.value].copy(), terms, float(ms.value)

    def percolator_register(self, queries: Sequence[np.ndarray], nterms: int, term_cost=None) -> dict:
        """registers the query set of this context's percolator (replacing any earlier one): query ids are indices into `queries`; term ids
        index a vocabulary of nterms terms; term_cost (e.g. document frequencies) only chooses the anchors"""
        arr, keep = _pack_queries(queries)
        cost = None if term_cost is None else _u32(term_cost)
        if cost is not None and len(cost) != nterms:
            raise TrinityError("term_cost needs one entry per vocabulary term")
        i = TrnPercolatorInfo()
        self._ck(self._L.trn_percolator_register(self._h, C.cast(arr, C.c_void_p), len(queries), nterms, _ptr(cost) if cost is not None else None,
                                                 C.byref(i)))
        self.percolator_info = {f: int(getattr(i, f)) for f, _ in TrnPercolatorInfo._fields_}
        return dict(self.percolator_info)

    def percolator_add(self, queries: Sequence[np.ndarray]) -> np.ndarray:
        """appends queries (trn_qnode trees over the registration's vocabulary) to the registered set; returns their ids (uint32, ascending
        from the info's next_id).  A refused call adds none of them."""
        arr, keep = _pack_queries(queries)
        i, first = TrnPercolatorInfo(), C.c_uint32()
        self._ck(self._L.trn_percolator_add(self._h, C.cast(arr, C.c_void_p) if len(queries) else None, len(queries), C.byref(first), C.byref(i)))
        self.percolator_info = {f: int(getattr(i, f)) for f, _ in TrnPercolatorInfo._fields_}
        return np.arange(first.value, first.value + len(queries), dtype=np.uint32)

    def percolator_remove(self, ids) -> dict:
        """removes live queries by id: no later percolate() returns them.  A refused call removes none of them."""
        a = _u32(ids).ravel()
        i = TrnPercolatorInfo()
        self._ck(self._L.trn_percolator_remove(self._h, _ptr(a) if len(a) else None, len(a), C.byref(i)))
        self.percolator_info = {f: int(getattr(i, f)) for f, _ in TrnPercolatorInfo._fields_}
        return dict(self.percolator_info)

    def percolator_last_update(self) -> dict:
        """device time (CUDA events around its uploads, copies and rebuild kernels) and host time of the last add / remove, ms"""
        dev, host = C.c_float(), C.c_float()
        self._ck(self._L.trn_percolator_last_update(self._h, C.byref(dev), C.byref(host)))
        return {"device_ms": float(dev.value), "host_ms": float(host.value)}

    def debug_percolator_registry(self):
        """the resident anchor index and unanchored list: (csr_off[nterms + 1], csr[entries, 2] of (query id, anchor ordinal), unanchored)"""
        nt, ne, nu = C.c_uint32(), C.c_uint64(), C.c_uint64()
        self._ck(self._L.trn_debug_percolator_registry(self._h, None, None, 0, None, 0, C.byref(nt), C.byref(ne), C.byref(nu)))
        off, csr, un = np.zeros(nt.value + 1, np.uint32), np.zeros((ne.value, 2), np.uint32), np.zeros(nu.value, np.uint32)
        self._ck(self._L.trn_debug_percolator_registry(self._h, _ptr(off), _ptr(csr), ne.value, _ptr(un), nu.value, C.byref(nt), C.byref(ne),
                                                       C.byref(nu)))
        return off, csr, un

    def percolate(self, docs: Sequence[np.ndarray]) -> "PercolationResult":
        """every registered query each document matches: docs are uint32 token arrays (EMPTY_TERM: a token outside the vocabulary)"""
        offs = np.zeros(len(docs) + 1, np.uint64)
        offs[1:] = np.cumsum([len(d) for d in docs])
        tok = _u32(np.concatenate([np.asarray(d, np.uint32) for d in docs]) if len(docs) else [])
        r = TrnPercolation()
        self._ck(self._L.trn_percolate(self._h, _ptr(offs), _ptr(tok) if len(tok) else None, len(docs), C.byref(r)))
        return PercolationResult(r)

    def index_documents(self, codec: int, docids, docs: Sequence[np.ndarray], nterms: int, positions: Optional[Sequence[np.ndarray]] = None,
                        payload_lens: Optional[Sequence[np.ndarray]] = None, payloads: Optional[Sequence[np.ndarray]] = None) -> "IndexedSegment":
        """== SegmentIndexSession begin / insert / commit for a batch: docs are uint32 term-id arrays (every id below nterms), docids their
        ids (any order, > 0, none twice); positions: per document the position of every token, None = token i at i + 1; payload_lens /
        payloads (both or neither): per document every token's payload size (0..8) and payload (uint64, the payload in its low bytes), as
        document_proxy::insert(term, pos, payload) takes them.  The inversion and the encode run on the device; the result holds the bytes
        commit() would have written."""
        d = _u32(docids)
        if len(d) != len(docs) or (positions is not None and len(positions) != len(docs)):
            raise TrinityError("index_documents: one docID (and one positions array) per document")
        if (payload_lens is None) != (payloads is None) or (payload_lens is not None and (len(payload_lens) != len(docs) or len(payloads) != len(docs))):
            raise TrinityError("index_documents: payload_lens and payloads come together, one array of each per document")
        offs = np.zeros(len(docs) + 1, np.uint64)
        offs[1:] = np.cumsum([len(x) for x in docs])
        tok = _u32(np.concatenate([np.asarray(x, np.uint32) for x in docs]) if len(docs) else [])
        pos = None
        if positions is not None:
            pos = _u32(np.concatenate([np.asarray(x, np.uint32) for x in positions]) if len(docs) else [])
            if len(pos) != len(tok):
                raise TrinityError("index_documents: one position per token")
        pl = pv = None
        if payload_lens is not None:
            pl = np.ascontiguousarray(np.concatenate([np.asarray(x, np.uint8) for x in payload_lens]) if len(docs) else np.zeros(0, np.uint8), np.uint8)
            pv = np.ascontiguousarray(np.concatenate([np.asarray(x, np.uint64) for x in payloads]) if len(docs) else np.zeros(0, np.uint64), np.uint64)
            if len(pl) != len(tok) or len(pv) != len(tok):
                raise TrinityError("index_documents: one payload length and one payload per token")
        return self.index_documents_flat(codec, d, offs, tok, nterms, pos, pl, pv)

    def index_documents_flat(self, codec: int, docids: np.ndarray, doc_offsets: np.ndarray, tokens: np.ndarray, nterms: int,
                             positions: Optional[np.ndarray] = None, payload_lens: Optional[np.ndarray] = None,
                             payloads: Optional[np.ndarray] = None) -> "IndexedSegment":
        """index_documents over the flat arrays of the C ABI (doc_offsets: uint64, ndocs + 1 entries; payload_lens uint8 and payloads
        uint64 one per token, both or neither)"""
        d, tok = _u32(docids), _u32(tokens)
        offs = np.ascontiguousarray(doc_offsets, np.uint64)
        pos = None if positions is None else _u32(positions)
        if (payload_lens is None) != (payloads is None):
            raise TrinityError("index_documents: payload_lens and payloads come together")
        r = TrnIndexed()
        if payload_lens is None:
            self._ck(self._L.trn_index_documents(self._h, codec, _ptr(d), _ptr(offs), _ptr(tok) if len(tok) else None,
                                                 _ptr(pos) if pos is not None and len(pos) else None, len(d), nterms, C.byref(r)))
        else:
            pl, pv = np.ascontiguousarray(payload_lens, np.uint8), np.ascontiguousarray(payloads, np.uint64)
            if len(pl) != len(tok) or len(pv) != len(tok):
                raise TrinityError("index_documents: one payload length and one payload per token")
            self._ck(self._L.trn_index_documents_payloads(self._h, codec, _ptr(d), _ptr(offs), _ptr(tok) if len(tok) else None,
                                                          _ptr(pos) if pos is not None and len(pos) else None, _ptr(pl) if len(pl) else None,
                                                          _ptr(pv) if len(pv) else None, len(d), nterms, C.byref(r)))
        return IndexedSegment(codec, r, d)

    def merge_sources(self, out_codec: int, sources: Sequence["MergeSource"], disable_optimizations: bool = False,
                      payloads: bool = False) -> "MergedSegment":
        """== MergeCandidatesCollection commit() + merge() into a fresh IndexSession of out_codec (trn_merge_sources): the sources fold
        newest generation first, each masked by the updated documents of the newer ones; the re-encoded terms run on the device.
        payloads=True (trn_merge_sources_payloads): re-encoded hits keep their payloads; without, such a hit is refused"""
        keep, arr = _merge_sources_c(sources)
        r = TrnMerged()
        f = self._L.trn_merge_sources_payloads if payloads else self._L.trn_merge_sources
        self._ck(f(self._h, out_codec, C.cast(arr, C.c_void_p) if len(sources) else None, len(sources), int(bool(disable_optimizations)), C.byref(r)))
        del keep
        return MergedSegment(out_codec, r, sources)

    def index_tokens(self, codec: int, docids, token_lists: Sequence[Sequence[str]], tdict: "TermDictionary") -> "IndexedSegment":
        """index_documents() with the tokens named: each resolved through the dictionary, whose size is nterms (an unknown name is refused)"""
        return self.index_documents(codec, docids, [np.array([tdict.term_id(t) for t in toks], np.uint32) for toks in token_lists], len(tdict))

    def close(self):
        if getattr(self, "_h", None):
            self._L.trn_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PercolationResult:
    """Percolator.percolate: per document the ascending ids of the registered queries it matches, the (document, query) pairs evaluated,
    the documents of the long launch and of the bitmap output, and the device times of both passes and the host time of the call"""

    def __init__(self, r: TrnPercolation):
        n, tot = int(r.ndocs), int(r.total)
        self.offsets = np.ctypeslib.as_array(r.offsets, shape=(n + 1,)).copy() if r.offsets else np.zeros(1, np.uint64)
        self.queries = np.ctypeslib.as_array(r.queries, shape=(tot,)).copy() if tot else np.zeros(0, np.uint32)
        self.ndocs, self.total, self.candidates = n, tot, int(r.candidates)
        self.long_docs, self.dense_docs = int(r.long_docs), int(r.dense_docs)
        self.count_ms, self.write_ms, self.total_ms = float(r.count_ms), float(r.write_ms), float(r.total_ms)

    def document(self, d: int) -> np.ndarray:
        return self.queries[int(self.offsets[d]): int(self.offsets[d + 1])]

    def __len__(self):
        return self.ndocs


class Percolator:
    """== Trinity's percolator_query::match (percolator.h) for a whole registered query set at once: which stored queries each incoming
    document matches.  queries: trn_qnode trees (parse_query); nterms: the size of the vocabulary their term ids index; term_cost: optional
    per-term cost (e.g. document frequency) that picks each query's anchors; source: a GpuIndexSource whose context to share (its index and
    exec_batch stay as they are), else a context of its own on `device`.  add() / remove() change the set in place: it then answers what
    registering the live queries fresh would, under the ids add() returned."""

    def __init__(self, queries: Sequence[np.ndarray], device: int = 0, nterms: int = 0, term_cost=None, source: Optional["GpuIndexSource"] = None):
        self.source = source if source is not None else GpuIndexSource(device)
        self._info = self.source.percolator_register(queries, nterms, term_cost)
        self._last = None

    def add(self, queries: Sequence[np.ndarray]) -> np.ndarray:
        """adds queries (parse_query trees over the registration's vocabulary) to the set; returns their new ids (uint32).  Ids are never
        reused; the vocabulary and term_cost stay the registration's."""
        ids = self.source.percolator_add(queries)
        self._info = dict(self.source.percolator_info)
        return ids

    def remove(self, ids) -> None:
        """removes queries by id; an id never issued, already removed or given twice is refused, and then none is removed"""
        self._info = self.source.percolator_remove(ids)

    def percolate(self, docs: Sequence[np.ndarray]) -> PercolationResult:
        self._last = self.source.percolate(docs)
        return self._last

    def percolate_tokens(self, token_lists: Sequence[Sequence[str]], tdict: "TermDictionary") -> PercolationResult:
        """percolate() with the tokens named: each resolved through the dictionary (an unknown name becomes EMPTY_TERM)"""
        return self.percolate([np.array([tdict.term_id(t) for t in toks], np.uint32) for toks in token_lists])

    def info(self) -> dict:
        return dict(self._info)

    def last_timings(self) -> dict:
        """device times (ms) of the count and write passes of the last percolate() call and its host time"""
        r = self._last
        return {} if r is None else {"count_ms": r.count_ms, "write_ms": r.write_ms, "total_ms": r.total_ms}

    def last_update_timings(self) -> dict:
        """device time (ms, CUDA events) and host time of the last add() / remove()"""
        return self.source.percolator_last_update()


def debug_percolator_plan(queries: Sequence[np.ndarray], nterms: int, term_cost=None):
    """the registration planner (csrc/percplan.h) on the host: per query (status, cover) with status 0 anchored, 1 unanchored, 2 cannot match
    and the anchor cover as ascending term ids"""
    arr, keep = _pack_queries(queries)
    cost = None if term_cost is None else _u32(term_cost)
    nq = len(queries)
    status, off = np.zeros(max(nq, 1), np.uint8), np.zeros(nq + 1, np.uint32)
    n = C.c_uint64()
    err = C.create_string_buffer(512)
    cap = 1 << 12
    while True:
        terms = np.zeros(cap, np.uint32)
        rc = lib().trn_debug_percolator_plan(C.cast(arr, C.c_void_p), nq, nterms, _ptr(cost) if cost is not None else None, _ptr(status), _ptr(off),
                                             _ptr(terms), cap, C.byref(n), err, 512)
        if rc == -6 and n.value > cap:
            cap = int(n.value)
            continue
        if rc != 0:
            raise TrinityError(f"rc={rc}: {err.value.decode()}")
        return [(int(status[q]), [int(t) for t in terms[int(off[q]): int(off[q + 1])]]) for q in range(nq)]


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


def segment_write(path: str, codec: int, index: np.ndarray, hits: Optional[np.ndarray], terms: np.ndarray, names: Sequence[str], field_statistics: dict,
                  updated_docids=()):
    """Writes the segment directory `path` (its last component a number, the generation) as Trinity's persist_segment / persist_terms do:
    index, hits.data (LUCENE), terms.data, terms.idx, id, and updated_documents.ids when there are updated (replaced or erased) docIDs.
    terms[i] <-> names[i]; terms without documents are left out.  Host code; Segment(path) and the reference's SegmentIndexSource open it."""
    index = np.ascontiguousarray(index, np.uint8)
    hits = np.zeros(0, np.uint8) if hits is None else np.ascontiguousarray(hits, np.uint8)
    terms = np.ascontiguousarray(terms, TERM_DTYPE)
    if len(names) != len(terms):
        raise TrinityError("segment_write: one name per term")
    enc = [n.encode("utf-8", "surrogateescape") if isinstance(n, str) else bytes(n) for n in names]
    arr = (C.c_char_p * len(enc))(*enc)
    upd = _u32(updated_docids)
    fs = field_statistics
    err = C.create_string_buffer(512)
    os.makedirs(os.path.dirname(os.path.abspath(str(path))), exist_ok=True)  # the C call creates the generation's directory itself
    rc = lib().trn_segment_write(str(path).encode(), codec, _ptr(index) if index.size else None, index.size, _ptr(hits) if hits.size else None, hits.size,
                                 _ptr(terms) if len(terms) else None, C.cast(arr, C.c_void_p) if len(enc) else None, len(terms), int(fs["sumTermHits"]),
                                 int(fs["totalTerms"]), int(fs["sumTermsDocs"]), int(fs["docsCnt"]), _ptr(upd) if len(upd) else None, len(upd), err, 512)
    if rc != 0:
        raise TrinityError(f"rc={rc}: {err.value.decode('utf-8', 'replace')}")


class IndexedSegment:
    """GpuIndexSource.index_documents: the index (and LUCENE hits.data) bytes of a batch of documents, the term_index_ctx tuple of every
    term id (documents == 0: the term has no posting), the field statistics commit() records, and the device times of the call."""

    def __init__(self, codec: int, r, docids: np.ndarray):
        self.codec = codec
        self.docids = docids.copy()  # of the batch, as given
        self.index = np.ctypeslib.as_array(r.index, shape=(int(r.index_bytes),)).copy() if r.index_bytes else np.zeros(0, np.uint8)
        self.hits = np.ctypeslib.as_array(r.hits, shape=(int(r.hits_bytes),)).copy() if r.hits_bytes else np.zeros(0, np.uint8)
        n = int(r.nterms)
        self.terms = np.ctypeslib.as_array(C.cast(r.terms, C.POINTER(C.c_uint8)), shape=(n * 12,)).view(TERM_DTYPE).copy()
        self.field_statistics = {"sumTermHits": int(r.sum_term_hits), "totalTerms": int(r.total_terms), "sumTermsDocs": int(r.sum_terms_docs),
                                 "docsCnt": int(r.docs_cnt)}
        self.max_docid = int(r.max_docid)
        self.sort_passes = int(r.sort_passes)
        self.timings = {"sort_ms": float(r.sort_ms), "postings_ms": float(r.postings_ms), "encode_ms": float(r.encode_ms), "total_ms": float(r.total_ms)}

    def write(self, path: str, names: Sequence[str], replaced=(), erased=()):
        """the segment directory of this batch: names[t] = the name of term id t; replaced = docIDs of this batch that older segments also
        hold, erased = docIDs deleted from older segments (both go to updated_documents.ids; an erased docID cannot be indexed here)"""
        both = np.intersect1d(self.docids, _u32(list(erased)))
        if len(both):
            raise TrinityError(f"IndexedSegment.write: docID {int(both[0])} is both indexed and erased (Already committed document)")
        segment_write(path, self.codec, self.index, self.hits, self.terms, names, self.field_statistics, list(replaced) + list(erased))

    def upload(self, gpu: "GpuIndexSource", names: Optional[Sequence[str]] = None):
        """uploads the index (the terms that have documents, in term-id order) and, for LUCENE, its hits; returns the term ids kept, or a
        TermDictionary of their names when names are given"""
        keep = np.flatnonzero(self.terms["documents"])
        gpu.upload(self.codec, self.index, self.terms[keep], self.max_docid)
        if self.codec == CODEC_LUCENE:
            gpu.upload_hits(self.index, self.hits)
        return keep if names is None else TermDictionary([names[int(t)] for t in keep])


@dataclass
class MergeSource:
    """one index source of a merge: its generation, index (and LUCENE hits.data) bytes, term tuples with their names in terms_cmp order
    (the order Segment exposes), and the docIDs it replaced or erased in older sources"""
    codec: int
    generation: int
    index: np.ndarray
    terms: np.ndarray
    names: Sequence[str]
    hits: Optional[np.ndarray] = None
    updated_docids: Optional[np.ndarray] = None

    @staticmethod
    def of_segment(seg: "Segment", path: str, generation: int) -> "MergeSource":
        hp = os.path.join(str(path), "hits.data")
        hits = np.fromfile(hp, np.uint8) if seg.codec == CODEC_LUCENE and os.path.exists(hp) else None
        if seg.codec == CODEC_LUCENE and hits is None:
            hits = np.zeros(0, np.uint8)
        return MergeSource(seg.codec, generation, seg.index, seg.terms, seg.names, hits, seg.masked_documents)


def _merge_sources_c(sources: Sequence[MergeSource]):
    """the trn_merge_source array and everything it points into (kept alive by the caller)"""
    keep = []
    arr = (TrnMergeSource * max(1, len(sources)))()
    for i, m in enumerate(sources):
        idx = np.ascontiguousarray(m.index, np.uint8)
        terms = np.ascontiguousarray(m.terms, TERM_DTYPE)
        if len(m.names) != len(terms):
            raise TrinityError(f"merge source {i}: one name per term")
        enc = [n.encode("utf-8", "surrogateescape") if isinstance(n, str) else bytes(n) for n in m.names]
        names = (C.c_char_p * max(1, len(enc)))(*enc)
        hits = None if m.hits is None else np.ascontiguousarray(m.hits, np.uint8)
        upd = _u32(np.zeros(0, np.uint32) if m.updated_docids is None else m.updated_docids)
        # a non-null pointer for an empty LUCENE hits.data: it is present, only empty
        hbuf = hits if hits is not None and hits.size else (np.zeros(1, np.uint8) if hits is not None else None)
        keep += [idx, terms, enc, names, hbuf, upd]
        arr[i] = TrnMergeSource(int(m.codec), int(m.generation), _ptr(idx) if idx.size else None, idx.size, _ptr(hbuf), 0 if hits is None else hits.size,
                                _ptr(terms) if len(terms) else None, C.cast(names, C.c_void_p) if len(enc) else None, len(terms),
                                _ptr(upd) if upd.size else None, upd.size)
    keep.append(arr)
    return keep, arr


def debug_merge_plan(out_codec: int, sources: Sequence[MergeSource], disable_optimizations: bool = False) -> dict:
    """the host planner of merge_sources (trn_debug_merge_plan; no GPU): candidate order, output terms with route / statistics flag /
    participants (candidate, term), the registries as (docID, newest candidate updating it), the GOOGLE countdown phase"""
    keep, arr = _merge_sources_c(sources)
    n = len(sources)
    T = sum(len(m.terms) for m in sources)
    U = sum(0 if m.updated_docids is None else len(m.updated_docids) for m in sources)
    order = np.zeros(max(1, n), np.uint32)
    route, stats = np.zeros(max(1, T), np.uint8), np.zeros(max(1, T), np.uint8)
    part_off, pc, pt = np.zeros(T + 1, np.uint32), np.zeros(max(1, T), np.uint32), np.zeros(max(1, T), np.uint32)
    ud, uf = np.zeros(max(1, U), np.uint32), np.zeros(max(1, U), np.uint32)
    nout, nparts, nupd, phase = C.c_uint32(), C.c_uint64(), C.c_uint64(), C.c_uint32()
    err = C.create_string_buffer(512)
    rc = lib().trn_debug_merge_plan(out_codec, C.cast(arr, C.c_void_p) if n else None, n, int(bool(disable_optimizations)), _ptr(order), _ptr(route),
                                    _ptr(stats), _ptr(part_off), _ptr(pc), _ptr(pt), C.byref(nout), C.byref(nparts), _ptr(ud), _ptr(uf), C.byref(nupd),
                                    C.byref(phase), err, 512)
    del keep
    if rc != 0:
        raise TrinityError(f"rc={rc}: {err.value.decode('utf-8', 'replace')}")
    k, q, u = nout.value, nparts.value, nupd.value
    return {"order": order[:n].tolist(), "route": route[:k].tolist(), "stats": stats[:k].tolist(), "part_off": part_off[:k + 1].tolist(),
            "parts": list(zip(pc[:q].tolist(), pt[:q].tolist())), "upd_docid": ud[:u].tolist(), "upd_first": uf[:u].tolist(),
            "countdown_phase": phase.value}


class MergedSegment:
    """GpuIndexSource.merge_sources: the merged index (and LUCENE hits.data), the output terms with their names, the field statistics
    (docsCnt: the distinct documents holding an output posting) and the phase times of the call"""

    def __init__(self, codec: int, r, sources: Sequence[MergeSource]):
        self.codec = codec
        self.index = np.ctypeslib.as_array(r.index, shape=(int(r.index_bytes),)).copy() if r.index_bytes else np.zeros(0, np.uint8)
        self.hits = np.ctypeslib.as_array(r.hits, shape=(int(r.hits_bytes),)).copy() if r.hits_bytes else np.zeros(0, np.uint8)
        n = int(r.nterms)
        if n:
            self.terms = np.ctypeslib.as_array(C.cast(r.terms, C.POINTER(C.c_uint8)), shape=(n * 12,)).view(TERM_DTYPE).copy()
            src, idx = np.ctypeslib.as_array(r.term_source, shape=(n,)), np.ctypeslib.as_array(r.term_index, shape=(n,))
            self.names = [sources[int(s)].names[int(t)] for s, t in zip(src, idx)]
        else:
            self.terms, self.names = np.zeros(0, TERM_DTYPE), []
        self.field_statistics = {"sumTermHits": int(r.sum_term_hits), "totalTerms": int(r.total_terms), "sumTermsDocs": int(r.sum_terms_docs),
                                 "docsCnt": int(r.docs_cnt)}
        self.counts = {"appended": int(r.appended), "reencoded": int(r.reencoded), "orphaned": int(r.orphaned), "postings_read": int(r.postings_read),
                       "postings_written": int(r.postings_written)}
        self.timings = {"decode_ms": float(r.decode_ms), "merge_ms": float(r.merge_ms), "encode_ms": float(r.encode_ms),
                        "assemble_ms": float(r.assemble_ms), "total_ms": float(r.total_ms)}

    def write(self, path: str):
        """the merged segment directory (its last component the generation); no updated_documents.ids: it masks nothing itself"""
        segment_write(path, self.codec, self.index, self.hits, self.terms, self.names, self.field_statistics)


RETAIN_ALL, RETAIN_DOCUMENT_IDS_UPDATES, RETAIN_DELETE = 0, 1, 2


def consider_tracked_sources(candidate_gens: Iterable[int], tracked_gens: Iterable[int]):
    """== MergeCandidatesCollection::consider_tracked_sources (merge.cpp:418-447): for every tracked generation, ascending, whether the
    application keeps its directory (RETAIN_ALL: not merged), keeps only its updated documents (RETAIN_DOCUMENT_IDS_UPDATES: merged, but an
    older tracked source that was not merged still needs them) or deletes it (RETAIN_DELETE)"""
    cands = set(int(g) for g in candidate_gens)
    out, last_not_candidate = [], None
    for i, g in enumerate(sorted(int(g) for g in tracked_gens)):
        if g not in cands:
            last_not_candidate = i
            out.append((g, RETAIN_ALL))
        elif last_not_candidate is not None:
            out.append((g, RETAIN_DOCUMENT_IDS_UPDATES))
        else:
            out.append((g, RETAIN_DELETE))
    return out
