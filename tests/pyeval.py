"""Pure-numpy evaluation of a trn_qnode tree with the reference's structural scoring rules
(docset_iterators_scorers.cpp:8-242).  TEST INFRASTRUCTURE: used to check the host query front-end / plan semantics on
CPU against the reference's exec_query, independent of any GPU."""
import numpy as np

import trinity_b200 as tb


def evaluate(nodes, lists, ndocs, weights=None, quirk=True, positions=None):
    """returns (match mask[ndocs+1], score[ndocs+1]) for node 0.  lists[t] = (docids, freqs); positions[t] = {docid: sorted positions}
    (only needed for PHRASE nodes)"""

    def rec(i):
        n = nodes[i]
        kind = int(n["kind"])
        if kind == tb.NODE_TERM:
            m = np.zeros(ndocs + 1, bool)
            s = np.zeros(ndocs + 1, np.float64)
            t = int(n["term"])
            if t != tb.EMPTY_TERM:
                d, f = lists[t]
                m[d] = True
                if weights is not None:
                    s[d] = [tb.bm25_score(float(n["weight"]), int(x) & 0xFFFF) for x in f]
            return m, s
        if kind == tb.NODE_PHRASE:
            # Phrase::consider_phrase_match (docset_iterators.cpp:66-158): every non-zero position p of the first term with term k at
            # p + k for all k counts as one match; score = score(matchCnt, sum of the terms' idf) (docset_iterators_scorers.cpp:195-228)
            m = np.zeros(ndocs + 1, bool)
            s = np.zeros(ndocs + 1, np.float64)
            ts = [int(nodes[int(n["first_child"]) + c]["term"]) for c in range(int(n["nchildren"]))]
            if any(t == tb.EMPTY_TERM for t in ts):
                return m, s
            docs = lists[ts[0]][0]
            for t in ts[1:]:
                docs = np.intersect1d(docs, lists[t][0], assume_unique=True)
            w = sum(float(nodes[int(n["first_child"]) + c]["weight"]) for c in range(int(n["nchildren"])))
            for d in docs:
                d = int(d)
                sets = [set(int(x) for x in positions[t][d]) for t in ts[1:]]
                cnt = sum(1 for p0 in positions[ts[0]][d] if p0 and all((int(p0) + k + 1) in sets[k] for k in range(len(sets))))
                if cnt:
                    m[d] = True
                    if weights is not None:
                        s[d] = tb.bm25_score(w, cnt & 0xFFFF)
            return m, s
        kids = [rec(int(n["first_child"]) + c) for c in range(int(n["nchildren"]))]
        if kind == tb.NODE_AND:
            m = np.logical_and.reduce([k[0] for k in kids])
            s = sum(k[1] for k in kids) * m
        elif kind == tb.NODE_OR:
            m = np.logical_or.reduce([k[0] for k in kids])
            s = sum(k[1] * k[0] for k in kids)
        elif kind == tb.NODE_NOT:
            m = kids[0][0] & ~kids[1][0]
            s = kids[0][1] * m
        elif kind == tb.NODE_SOME:  # DisjunctionSome: >= min children match; the matching children score
            m = sum(k[0].astype(np.int32) for k in kids) >= int(n["term"])
            s = sum(k[1] * k[0] for k in kids)
        else:  # OPTIONAL
            m = kids[0][0]
            s = (kids[0][1] + kids[1][1] * kids[1][0]) * m
        return m, s * m

    def cost(i):
        n = nodes[i]
        kind = int(n["kind"])
        if kind == tb.NODE_TERM:
            t = int(n["term"])
            return 0 if t == tb.EMPTY_TERM else len(lists[t][0])
        kids = [cost(int(n["first_child"]) + c) for c in range(int(n["nchildren"]))]
        if kind == tb.NODE_PHRASE:
            return min(kids)
        if kind in (tb.NODE_NOT, tb.NODE_OPTIONAL):
            return kids[0]
        if kind == tb.NODE_SOME:
            return sum(sorted(kids)[:max(0, len(kids) - int(n["term"]) + 1)])
        return min(kids) if kind == tb.NODE_AND else sum(kids)

    # the reference's root-Filter-over-disjunction quirk (exec.cpp:488-501 + docset_spans.cpp:98-111), see planner.cpp
    root, traversed = 0, False
    while int(nodes[root]["kind"]) == tb.NODE_NOT and cost(int(nodes[root]["first_child"]) + 1) <= cost(int(nodes[root]["first_child"])):
        root, traversed = int(nodes[root]["first_child"]), True
    if not (quirk and traversed and int(nodes[root]["kind"]) == tb.NODE_OR):
        root = 0
    return rec(root)
