"""Percolator (test infrastructure): the query lists the percolator is checked on, seeded documents, a Python evaluator of a query tree on
a token sequence (the registry's meaning), a Python restatement of the registry's anchor-cover rules (csrc/percplan.h) and the ctypes
wrapper of the reference oracle (oracle/_ref/libtrinity_ref_perc.so: the reference's own percolator_query::match)."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

import trinity_b200 as tb

ROOT = Path(__file__).resolve().parent.parent
PERC_SO = ROOT / "oracle" / "_ref" / "libtrinity_ref_perc.so"
EMPTY = tb.EMPTY_TERM

# the percolator vocabulary of the tests: t1..t12 (the exec tests' names) and w1..w9 (the phrase tests' names)
VOCAB = [f"t{i}" for i in range(1, 13)] + [f"w{i}" for i in range(1, 10)]


def query_lists():
    """[(text, parser flags, MatchSome min or 0)]: every query list the exec tests use, with the reference parser flags they need"""
    from test_frontend_cpu import EXTRA, OPTIONAL_QUERIES, SOME_QUERIES
    from test_gpu_masked import QUERIES as MASKED
    from test_gpu_parity import TEMPLATES
    from test_gpu_segments import QUERIES as SEGMENTS
    from test_gpu_sharded import DOCS_QUERIES
    from test_phrase_cpu import QUERIES as PHRASES
    flags = (lambda q: (8 if "<" in q else 0) | (16 if "[" in q else 0))
    return [(q, flags(q), 0) for q in TEMPLATES + EXTRA + MASKED + SEGMENTS + DOCS_QUERIES + PHRASES + OPTIONAL_QUERIES] + [(q, 16, m) for q, m in SOME_QUERIES]


# shapes the percolator tests add: phrases with repeated terms, out-of-vocabulary phrase terms, MatchSome at min 1, n and above n
EXTRA_SHAPES = [('"w1 w1"', 0, 0), ('"w1 w1 w1"', 0, 0), ('"w1 oov1"', 0, 0), ('"oov1 w1"', 0, 0), ('"w1 w2 w1 w2"', 0, 0), ('t1 "w1 w2"', 0, 0),
                ('"w3 w4" OR "w4 w3"', 0, 0), ('t1 NOT "w1 w2"', 0, 0), ("[t1, t2, t3]", 16, 1), ("[t1, t2, t3]", 16, 3), ("[t1, t2, t3]", 16, 4),
                ('[t1, "w1 w2", t3 AND t4]', 16, 2), ("[t1, oov1, t2]", 16, 2), ("[oov1, oov2]", 16, 1), ("t1 <t2 OR t3>", 8, 0),
                ("t1 <oov1>", 8, 0), ('"w1 w2 w3 w4 w5 w6 w7 w8 w9 w1 w2 w3 w4 w5 w6 w7"', 0, 0), ("t1 AND t1", 0, 0),
                ("(t1 OR t2) NOT (t2 OR t3)", 0, 0)]
# (the reference's parser refuses "t1 NOT t1": not comparable)

# the "check first" shapes: const-true expressions that do not stand beside a conjunction operand.  The front-end drops their <...>
# wrapper (`<t1>` parses to `t1`), so the tree means the exec_query meaning, while the reference's percolator evaluates
# consttrueexpr as true.  A tree cannot say which it came from, so the registry takes the tree's meaning (pinned in
# test_percolate_cpu); a leading NOT does not parse in the front-end.
CONST_TRUE_SHAPES = [("<t1>", 8, 0), ("t1 OR <t2>", 8, 0), ("<t1> OR <t2>", 8, 0), ("[<t1>, t2]", 24, 1), ("<t1> NOT t2", 8, 0)]


def random_docs(rng, n, vocab=len(VOCAB), max_len=40, oov=0.1, lens=None):
    """n token arrays: lengths uniform in 0..max_len (or `lens`), tokens Zipf-like over the vocabulary, a share `oov` outside it"""
    p = 1.0 / np.arange(1, vocab + 1)
    p /= p.sum()
    out = []
    for i in range(n):
        L = int(lens[i]) if lens is not None else int(rng.integers(0, max_len + 1))
        t = rng.choice(vocab, size=L, p=p).astype(np.uint32)
        t[rng.random(L) < oov] = EMPTY
        out.append(t)
    return out


def tokens_of(names, tdict):
    return np.array([tdict.term_id(s) for s in names], np.uint32)


# ------------------------------------------------------------------------------------------------ the registry's meaning
def evaluate(nodes, doc, i=0):
    """does the tree (trn_qnode array, root 0) match the token sequence `doc` under the percolator's proxy: a term is on the document
    when a token equals it; a phrase when its terms stand at consecutive positions; EMPTY_TERM never equals anything"""
    x = nodes[i]
    k, f, n = int(x["kind"]), int(x["first_child"]), int(x["nchildren"])
    if k == tb.NODE_TERM:
        t = int(x["term"])
        return t != EMPTY and bool(np.any(doc == t))
    if k == tb.NODE_PHRASE:
        ts = [int(nodes[f + j]["term"]) for j in range(n)]
        if EMPTY in ts or len(doc) < n:
            return False
        hit = np.ones(len(doc) - n + 1, bool)
        for j, t in enumerate(ts):
            hit &= doc[j: len(doc) - n + 1 + j] == t
        return bool(hit.any())
    kids = [evaluate(nodes, doc, f + j) for j in range(n)]
    if k == tb.NODE_AND:
        return all(kids)
    if k == tb.NODE_OR:
        return any(kids)
    if k == tb.NODE_NOT:
        return kids[0] and not any(kids[1:])
    if k == tb.NODE_OPTIONAL:
        return kids[0]
    if k == tb.NODE_SOME:
        m = int(x["term"])
        return m >= 1 and sum(kids) >= m
    raise ValueError(k)


# ------------------------------------------------------------------------------------------------ anchor covers (csrc/percplan.h)
NEVER, UNANCHORED = "never", "unanchored"


def cover(nodes, cost, i=0):
    """(kind, terms, cost): NEVER (no document matches), UNANCHORED (a match may hold no term) or ("set", sorted terms every match holds
    one of, their summed cost)"""
    x = nodes[i]
    k, f, n = int(x["kind"]), int(x["first_child"]), int(x["nchildren"])
    c = (lambda t: 1 if cost is None else int(cost[t]))
    if k == tb.NODE_TERM:
        t = int(x["term"])
        return (NEVER, (), 0) if t == EMPTY else ("set", (t,), c(t))
    if k == tb.NODE_PHRASE:
        ts = [int(nodes[f + j]["term"]) for j in range(n)]
        if EMPTY in ts:
            return (NEVER, (), 0)
        t = min(ts, key=lambda t: (c(t), t))
        return ("set", (t,), c(t))
    kids = [cover(nodes, cost, f + j) for j in range(n)]
    if k in (tb.NODE_NOT, tb.NODE_OPTIONAL):
        return kids[0]
    if k == tb.NODE_AND:
        if any(kd[0] == NEVER for kd in kids):
            return (NEVER, (), 0)
        sets = [kd for kd in kids if kd[0] == "set"]
        return min(sets, key=lambda kd: (kd[2], kd[1])) if sets else (UNANCHORED, (), 0)
    live = [kd for kd in kids if kd[0] != NEVER]
    if k == tb.NODE_OR:
        need = len(live)
        if not live:
            return (NEVER, (), 0)
    else:  # SOME: of the children that can match, any len - min + 1 hold one true child
        m = int(x["term"])
        if m < 1 or m > len(live):
            return (NEVER, (), 0)
        need = len(live) - m + 1
    order = sorted(range(len(live)), key=lambda j: (live[j][0] != "set", live[j][2], live[j][1], j))[:need]
    if any(live[j][0] != "set" for j in order):
        return (UNANCHORED, (), 0)
    ts = sorted(set(t for j in order for t in live[j][1]))
    return ("set", tuple(ts), sum(c(t) for t in ts))


# ------------------------------------------------------------------------------------------------ the reference oracle
def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class RefPercolator:
    """percolator_query(q).match(proxy) for every (document, query) pair, on one host thread"""

    def __init__(self, queries, vocab=VOCAB):
        """queries: [(text, parser flags, MatchSome min or 0)]"""
        if not PERC_SO.exists():
            raise RuntimeError(f"{PERC_SO} missing: run oracle/build_percolate.sh (build() does)")
        L = self.L = C.CDLL(str(PERC_SO))
        vp, u32 = C.c_void_p, C.c_uint32
        L.tperc_last_error.restype = C.c_char_p
        L.tperc_new.restype = vp
        L.tperc_new.argtypes = [vp, vp, vp, u32, vp, u32]
        L.tperc_free.argtypes = [vp]
        L.tperc_run.restype = C.c_int64
        L.tperc_run.argtypes = [vp, vp, vp, u32]
        L.tperc_last.argtypes = [vp, vp, vp]
        qs = [q.encode() for q, _, _ in queries] or [b""]
        qa = (C.c_char_p * len(qs))(*qs)
        fl = np.array([f for _, f, _ in queries] or [0], np.uint32)
        mn = np.array([m for _, _, m in queries] or [0], np.uint32)
        vs = [v.encode() for v in vocab] or [b""]
        va = (C.c_char_p * len(vs))(*vs)
        h = L.tperc_new(C.cast(qa, vp), _p(fl), _p(mn), len(queries), C.cast(va, vp), len(vocab))
        if not h:
            raise RuntimeError(L.tperc_last_error().decode())
        self.h = C.c_void_p(h)

    def run(self, docs):
        """-> per document the ascending ids of the queries it matches"""
        offs = np.zeros(len(docs) + 1, np.uint64)
        offs[1:] = np.cumsum([len(d) for d in docs])
        tok = np.ascontiguousarray(np.concatenate(docs) if docs else np.zeros(0), np.uint32)
        n = self.L.tperc_run(self.h, _p(offs), _p(tok) if tok.size else None, len(docs))
        if n < 0:
            raise RuntimeError(self.L.tperc_last_error().decode())
        o, ids = np.zeros(len(docs) + 1, np.uint64), np.zeros(max(n, 1), np.uint32)
        self.L.tperc_last(self.h, _p(o), _p(ids))
        return [ids[int(o[d]): int(o[d + 1])].copy() for d in range(len(docs))]

    def __del__(self):
        try:
            self.L.tperc_free(self.h)
        except Exception:
            pass
