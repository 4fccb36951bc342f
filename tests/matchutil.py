"""Test infrastructure of the default exec mode (TRN_MODE_MATCHED_TERMS): the reference harness oracle/_ref/libtrinity_ref_matches.so
(oracle/ref_matches.cpp: indexes built by the reference Encoders with payloads, exec_query with no ExecFlags), corpora with payloads, and a
numpy restatement of queryexec_ctx::collect_doc_matching_terms (queryexec_ctx.cpp:382-648)."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

import trinity_b200 as tb
from pyeval import evaluate

SO = Path(__file__).resolve().parent.parent / "oracle" / "_ref" / "libtrinity_ref_matches.so"
_lib = None


def load_matches():
    global _lib
    if _lib is None:
        if not SO.exists():
            raise RuntimeError(f"{SO} missing: run __graft_entry__.build() (oracle/build_matches.sh)")
        L = C.CDLL(str(SO))
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        for name, res, args in [
            ("trefm_last_error", C.c_char_p, []), ("trefm_new", vp, [C.c_int]), ("trefm_free", None, [vp]),
            ("trefm_add_term", C.c_int, [vp, C.c_char_p, vp, vp, u32, vp, vp, vp]), ("trefm_finish", C.c_int, [vp, u64]),
            ("trefm_index_size", u64, [vp]), ("trefm_index_data", vp, [vp]), ("trefm_hits_size", u64, [vp]), ("trefm_hits_data", vp, [vp]),
            ("trefm_term", None, [vp, u32, C.POINTER(u32), C.POINTER(u32), C.POINTER(u32)]),
            ("trefm_exec_matches", C.c_int64, [vp, C.c_char_p, u32, u32, vp, u32]),
            ("trefm_last", None, [vp] + [C.POINTER(vp)] * 7 + [C.POINTER(u64), C.POINTER(u64)]),
        ]:
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data if a.size else None


class RefMatches:
    """one in-memory index built through the reference's own Encoder, hits with payloads"""

    def __init__(self, codec: int):
        self.L = load_matches()
        self.codec = codec
        self.h = self.L.trefm_new(codec)
        self.n = 0

    def add_term(self, name, docids, freqs, positions, plens, payloads):
        d, f = np.ascontiguousarray(docids, np.uint32), np.ascontiguousarray(freqs, np.uint32)
        p, pl, pv = np.ascontiguousarray(positions, np.uint32), np.ascontiguousarray(plens, np.uint8), np.ascontiguousarray(payloads, np.uint64)
        rc = self.L.trefm_add_term(self.h, name.encode(), _ptr(d), _ptr(f), len(d), _ptr(p), _ptr(pl), _ptr(pv))
        assert rc >= 0, self.L.trefm_last_error().decode()
        self.n += 1

    def finish(self, ndocs):
        assert self.L.trefm_finish(self.h, ndocs) == 0, self.L.trefm_last_error().decode()

    def index(self):
        n = self.L.trefm_index_size(self.h)
        return np.ctypeslib.as_array((C.c_uint8 * n).from_address(self.L.trefm_index_data(self.h))).copy() if n else np.zeros(0, np.uint8)

    def hits(self):
        n = self.L.trefm_hits_size(self.h)
        return np.ctypeslib.as_array((C.c_uint8 * n).from_address(self.L.trefm_hits_data(self.h))).copy() if n else np.zeros(0, np.uint8)

    def terms(self):
        out = np.zeros(self.n, tb.TERM_DTYPE)
        for i in range(self.n):
            a, b, c = C.c_uint32(), C.c_uint32(), C.c_uint32()
            self.L.trefm_term(self.h, i, C.byref(a), C.byref(b), C.byref(c))
            out[i] = (a.value, b.value, c.value)
        return out

    def exec(self, q: str, parser_flags: int = 0, min_match: int = 0, masked=()):
        """consider(const matched_document &) stream: [(docid, [(term, freq, positions, payload_lens, payloads)] by ascending term)]"""
        m = np.ascontiguousarray(list(masked), np.uint32)
        n = self.L.trefm_exec_matches(self.h, q.encode(), parser_flags, min_match, _ptr(m), len(m))
        assert n >= 0, self.L.trefm_last_error().decode()
        ps = [C.c_void_p() for _ in range(7)]
        nt, nh = C.c_uint64(), C.c_uint64()
        self.L.trefm_last(self.h, *[C.byref(p) for p in ps], C.byref(nt), C.byref(nh))

        def arr(p, ct, cnt, dt):
            return np.ctypeslib.as_array((ct * cnt).from_address(p.value)).astype(dt) if cnt else np.zeros(0, dt)
        docs, tc = arr(ps[0], C.c_uint32, n, np.uint32), arr(ps[1], C.c_uint32, n, np.uint32)
        terms, freqs = arr(ps[2], C.c_uint32, nt.value, np.uint32), arr(ps[3], C.c_uint32, nt.value, np.uint32)
        pay, pos, pl = arr(ps[4], C.c_uint64, nh.value, np.uint64), arr(ps[5], C.c_uint16, nh.value, np.uint16), arr(ps[6], C.c_uint8, nh.value, np.uint8)
        out, ti, hi = [], 0, 0
        for i in range(n):
            ts = []
            for _ in range(int(tc[i])):
                f = int(freqs[ti])
                ts.append((int(terms[ti]), f, pos[hi:hi + f], pl[hi:hi + f], pay[hi:hi + f]))
                ti += 1
                hi += f
            out.append((int(docs[i]), sorted(ts, key=lambda x: x[0])))
        return out

    def __del__(self):
        if getattr(self, "h", None):
            self.L.trefm_free(self.h)
            self.h = None


def payload_hits(rng, n, change=0.35):
    """n hits' payload sizes (0..8, a size persists with probability 1 - change: sizes grow and shrink inside a document) and values"""
    sizes = np.zeros(n, np.uint8)
    s = int(rng.integers(0, 9))
    for i in range(n):
        if rng.random() < change:
            s = int(rng.integers(0, 9))
        sizes[i] = s
    vals = rng.integers(0, 1 << 63, size=n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=n, dtype=np.uint64)
    mask = np.array([(1 << (8 * int(x))) - 1 if x < 8 else (1 << 64) - 1 for x in sizes], np.uint64)
    return sizes, vals & mask


def doc_corpus(rng, ndocs, vocab, doclen=(3, 30), first_doc=1):
    """document-major text: per document a run of tokens (Zipf over `vocab` terms) at positions 1, 2, ...; every hit carries a payload.
    -> lists[t] = (docids, freqs, positions, payload sizes, payloads), positions[t] = {docid: [positions]}"""
    prob = 1.0 / np.arange(1, vocab + 1)
    prob /= prob.sum()
    per = [dict() for _ in range(vocab)]
    for d in range(first_doc, first_doc + ndocs):
        toks = rng.choice(vocab, size=int(rng.integers(doclen[0], doclen[1] + 1)), p=prob)
        for pos, t in enumerate(toks, start=1):
            per[int(t)].setdefault(d, []).append(pos)
    return lists_from(rng, per)


def lists_from(rng, per):
    lists, positions = [], []
    for t in range(len(per)):
        docs = np.array(sorted(per[t]), np.uint32)
        freqs = np.array([len(per[t][int(d)]) for d in docs], np.uint32)
        pos = np.array([p for d in docs for p in per[t][int(d)]], np.uint32)
        sz, pv = payload_hits(rng, len(pos))
        lists.append((docs, freqs, pos, sz, pv))
        positions.append({int(d): per[t][int(d)] for d in docs})
    return lists, positions


def host_build(codec, lists):
    """the same postings through the host IndexBuilder (streaming, with payloads) -> (index, hits, terms)"""
    b = tb.IndexBuilder(codec)
    for docs, freqs, pos, sz, pv in lists:
        b.begin_term()
        h = 0
        for d, f in zip(docs.tolist(), freqs.tolist()):
            b.begin_document(d)
            for _ in range(f):
                b.new_hit(int(pos[h]), int(pv[h]).to_bytes(8, "little")[: int(sz[h])])
                h += 1
            b.end_document()
        b.end_term()
    return b.index(), b.hits(), b.terms_array()


def ref_build(codec, lists, names, ndocs):
    r = RefMatches(codec)
    for n, (docs, freqs, pos, sz, pv) in zip(names, lists):
        r.add_term(n, docs, freqs, pos, sz, pv)
    r.finish(ndocs)
    return r


def restated_terms(nodes, lists, positions, ndocs):
    """numpy restatement: the matches of node 0 in the default exec mode (no root-filter quirk) and per match the set of terms
    collect_doc_matching_terms reports -> {docid: frozenset(term)}"""
    pl = [(l[0], l[1]) for l in lists]
    memo = {}

    def ev(i):
        if i not in memo:
            memo[i] = _eval_at(nodes, pl, ndocs, positions, i)
        return memo[i]

    def collect(i, d):
        n = nodes[i]
        k = int(n["kind"])
        fc, nc = int(n["first_child"]), int(n["nchildren"])
        if k == tb.NODE_TERM:
            return {int(n["term"])}
        if k == tb.NODE_PHRASE:
            return {int(nodes[fc + c]["term"]) for c in range(nc)}
        if k == tb.NODE_AND:
            return set().union(*[collect(fc + c, d) for c in range(nc)])
        if k in (tb.NODE_OR, tb.NODE_SOME):
            return set().union(*[collect(fc + c, d) for c in range(nc) if ev(fc + c)[d]])
        if k == tb.NODE_NOT:
            return collect(fc, d)
        if k == tb.NODE_OPTIONAL:
            s = collect(fc, d)
            return s | collect(fc + 1, d) if ev(fc + 1)[d] else s
        raise AssertionError(k)

    root = ev(0)
    return {int(d): frozenset(collect(0, int(d))) for d in np.flatnonzero(root)}


def _eval_at(nodes, lists, ndocs, positions, i):
    """evaluate() of the subtree at node i: the node array re-rooted at i (children keep their relative layout)"""
    sub = nodes[i:].copy()
    for j in range(len(sub)):
        if int(sub[j]["kind"]) not in (tb.NODE_TERM,) and int(sub[j]["nchildren"]):
            sub[j]["first_child"] = int(sub[j]["first_child"]) - i
    return evaluate(sub, lists, ndocs, quirk=False, positions=positions)[0]


def gpu_as_list(res, q):
    return [(d, [(t, f, p, l, v) for t, f, p, l, v in ts]) for d, ts in res.matches(q)]


def assert_same_matches(got, want, what):
    """docIDs, term sets, freqs and every hit's (pos, payload_len, payload) bit for bit"""
    assert len(got) == len(want), f"{what}: {len(got)} matches, the reference has {len(want)}"
    for (gd, gt), (wd, wt) in zip(got, want):
        assert gd == wd, f"{what}: docID {gd} where the reference has {wd}"
        assert [t[0] for t in gt] == [t[0] for t in wt], f"{what}: doc {gd}: terms {[t[0] for t in gt]} vs reference {[t[0] for t in wt]}"
        for (t, f, p, l, v), (_, wf, wp, wl, wv) in zip(gt, wt):
            assert f == wf, f"{what}: doc {gd} term {t}: freq {f} vs {wf}"
            assert np.array_equal(np.asarray(p, np.uint16), wp), f"{what}: doc {gd} term {t}: positions {p} vs {wp}"
            assert np.array_equal(np.asarray(l, np.uint8), wl), f"{what}: doc {gd} term {t}: payload lengths {l} vs {wl}"
            assert np.array_equal(np.asarray(v, np.uint64), wv), f"{what}: doc {gd} term {t}: payloads {v} vs {wv}"
