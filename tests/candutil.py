"""Host-side restatements of the candidate-driven conjunction (exec_docs_cand.cuh) and the corpora that reach its switch points
(test infrastructure, no GPU):
  * lead_block_forms: how google_block_to_array decodes every block of a lead — the code lengths of its doc deltas and where, and why,
    the in-slot loop over the 80 staged bytes stops;
  * probe_forms: how cand_exec_google decides every candidate against one probed term — out of range, the block-last hit without a
    gather, the walk of google_block_find (dp4a groups, 1- and 2-byte steps, the spill to global memory on longer codes), the bitmap
    probe of a term with a resident bitmap, and the sparse docID -> block table's boundaries;
  * eval_sets: a plain evaluator of a query tree over sorted docID arrays (no per-docID mask, so it reaches docID 2^32 - 2);
  * probe_order: the planner's probe order (plan_batch: the rarest necessary term leads, the other necessary terms rarest first, then
    the rest rarest first), from the terms' block counts;
  * seeded corpus builders for test_candidates_cpu and test_gpu_candidate_edges."""
from __future__ import annotations

from collections import Counter

import numpy as np

import trinity_b200 as tb

G = tb.CODEC_GOOGLE
GATHER = 80  # kGatherBytes: staged bytes per lane, from the 16-byte-aligned address below the first doc-delta byte
DENSE_ALIGN = 17  # kDenseAlignShift: a resident bitmap starts at first_doc rounded down to 2^17
TOP = 2**32 - 2  # the largest docID (2^32 - 1 is kCandInvalid / DocIDsEND)


def vb_len(b0: int) -> int:
    return 1 if b0 < 0x80 else 2 if b0 < 0xC0 else 3 if b0 < 0xE0 else 4 if b0 < 0xF0 else 5


def vb_get(buf, p: int):
    """(value, next p) of the prefix-varbyte code at buf[p] (varbyte.h)"""
    b0 = int(buf[p])
    if b0 < 0x80:
        return b0, p + 1
    if b0 < 0xC0:
        return ((b0 & 0x3F) << 8) | int(buf[p + 1]), p + 2
    if b0 < 0xE0:
        return ((b0 & 0x1F) << 16) | int(buf[p + 1]) | (int(buf[p + 2]) << 8), p + 3
    if b0 < 0xF0:
        return ((b0 & 0x0F) << 24) | (int(buf[p + 1]) << 16) | (int(buf[p + 2]) << 8) | int(buf[p + 3]), p + 4
    return int(buf[p + 1]) | (int(buf[p + 2]) << 8) | (int(buf[p + 3]) << 16) | (int(buf[p + 4]) << 24), p + 5


def term_tuple(terms, t: int):
    return tuple(int(x) for x in terms[t])


class Blocks:
    """a term's blocks as the kernel sees them: the directory (blk_last, blk_off, block sizes) and every block's doc-delta codes"""

    def __init__(self, index, term):
        last, off, first = tb.directory_probe(G, index, term)
        self.nb = len(last) - 1 if len(last) else 0
        self.docs, self.first = int(term[0]), int(first)
        self.last = [int(x) for x in last[: self.nb]]
        self.off = [int(x) for x in off[: self.nb]]
        self.n = [32 if b + 1 < self.nb else self.docs - 32 * (self.nb - 1) for b in range(self.nb)]
        self.codes = []  # per block: [(value, length)] of its n - 1 doc deltas
        for b in range(self.nb):
            p, cs = self.off[b], []
            for _ in range(self.n[b] - 1):
                v, q = vb_get(index, p)
                cs.append((v, q - p))
                p = q
            self.codes.append(cs)

    def prev(self, b):
        return self.last[b - 1] if b else 0

    def block_docs(self, b):
        d, out = self.prev(b), []
        for v, _ in self.codes[b]:
            d += v
            out.append(d)
        return out + [self.last[b]]


def lead_block_forms(index, term):
    """per block of the term: dict(b, n, mis, lens, stop, why, edge) — `stop` is the number of doc deltas google_block_to_array decodes
    inside its 80-byte slot; `why` the reason it stops there: "end" (all n - 1 deltas), "slot" (the next code could end past byte 80)
    or "long" (the next code is 4 or 5 bytes); `edge` is 80 when a 3-byte code ends exactly on slot byte 80 inside the slot, 81 when
    the loop stops at a 3-byte code that would end one byte past it, else None"""
    B = Blocks(index, term)
    out = []
    for b in range(B.nb):
        mis = B.off[b] & 15
        lens = [L for _, L in B.codes[b]]
        p, i, why, edge = 0, 0, "end", None
        while i < len(lens):
            if mis + p + 3 > GATHER:
                why = "slot"
                if lens[i] == 3 and mis + p + 3 == GATHER + 1:
                    edge = 81
                break
            if lens[i] >= 4:
                why = "long"
                break
            if lens[i] == 3 and mis + p + 3 == GATHER:
                edge = 80
            p += lens[i]
            i += 1
        out.append(dict(b=b, n=B.n[b], mis=mis, lens=lens, stop=i, why=why, edge=edge))
    return out


def block_find(codes, prev, target):
    """google_block_find over one block's doc-delta codes [(value, length)] -> (hit, how): how is ("dp4a_eq" | "dp4a_gt", 1) when a
    dp4a group's sum reached the target (equal / above) and the 1-byte step after it decided, ("step", L) when a 1- or 2-byte step
    decided, ("spill", L) when a code of L >= 3 bytes sent the walk to global memory and it decided there, ("end", L) when the deltas
    ran out below the target (L: the spill's code length, 0 without one)"""
    nd, doc, i, spill = len(codes), prev, 0, 0
    while i < nd and not spill:
        group = None
        while i + 4 <= nd:
            four = codes[i: i + 4]
            if any(L != 1 for _, L in four):
                break
            s = sum(v for v, _ in four)
            if doc + s >= target:
                group = "dp4a_eq" if doc + s == target else "dp4a_gt"
                break
            doc += s
            i += 4
        for _ in range(4):
            if i >= nd:
                break
            v, L = codes[i]
            if L >= 3:
                spill = L
                break
            doc += v
            i += 1
            if doc >= target:
                return doc == target, ((group, 1) if group else ("step", L))
    while i < nd:
        doc += codes[i][0]
        i += 1
        if doc >= target:
            return doc == target, ("spill", spill)
    return False, ("end", spill)


def probe_forms(index, term, candidates, dense=False, lookup=True):
    """(hits, forms): per candidate whether cand_exec_google finds it in the term, and a Counter of the forms its probes take (see the
    module docstring).  dense: the term has a resident bitmap.  The block each candidate goes to is the one tb.directory_lookup (the
    kernels' own lookup code) returns; lookup=False skips that call (the caller checked it)"""
    cands = np.asarray(candidates, np.uint64)
    B = Blocks(index, term)
    forms, hits = Counter(), np.zeros(len(cands), bool)
    if B.nb == 0:
        return hits, forms
    lastd = B.last[-1]
    if dense:
        base = (B.first >> DENSE_ALIGN) << DENSE_ALIGN
        end = (((lastd >> DENSE_ALIGN) + 1) << DENSE_ALIGN) - 1
        docs = set(int(x) for b in range(B.nb) for x in B.block_docs(b))
        for k, c in enumerate(int(x) for x in cands):
            hits[k] = c in docs
            forms["bm_low" if c < B.first else "bm_high" if c > lastd else "bm_in"] += 1
            for name, at in (("bm_first", B.first), ("bm_last", lastd), ("bm_base", base), ("bm_end", end)):
                if c == at:
                    forms[name] += 1
        return hits, forms
    if lookup:
        blocks, tf_shift, _ = tb.directory_lookup(G, index, term, cands.astype(np.uint32))
    else:
        blocks, tf_shift = None, 32
    forms["table" if tf_shift < 32 else "no_table"] += len(cands)
    for k, c in enumerate(int(x) for x in cands):
        if c > lastd:
            forms["above_last"] += 1
            continue
        lo = int(np.searchsorted(np.asarray(B.last, np.uint64), c, "left"))
        assert blocks is None or int(blocks[k]) == lo, (c, int(blocks[k]), lo)
        if tf_shift < 32 and B.first < c and c & ((1 << tf_shift) - 1) == 0:
            forms["tf_edge"] += 1
        if B.last[lo] == c:
            hits[k] = True
            forms["block_last"] += 1
            continue
        prev = B.prev(lo)
        if c < B.first:
            forms["below_first"] += 1
        elif lo and c == prev + 1:
            forms["prev_plus_1"] += 1
        if lo and c < B.block_docs(lo)[0]:
            forms["between_blocks"] += 1
        hit, (how, L) = block_find(B.codes[lo], prev, c)
        hits[k] = hit
        forms[f"{how}{L}_{'hit' if hit else 'miss'}"] += 1
    return hits, forms


def probe_targets(index, term, dense=False):
    """docIDs that put a probe of the term at each of its switch points: its first and last docID and one outside each, every block's
    last docID and the one after it, the docIDs around every dp4a group's sum and behind every code of 2 or more bytes, the table's
    boundaries, and (dense) the 2^17-aligned ends of the bitmap's span"""
    B = Blocks(index, term)
    out = {B.first, B.first - 1, B.last[-1], B.last[-1] + 1}
    for b in range(B.nb):
        out |= {B.last[b], B.last[b] + 1}
        if dense:
            continue
        docs = B.block_docs(b)
        for i, (v, L) in enumerate(B.codes[b]):
            if L >= 2:
                out |= {docs[i], docs[i] - 1}
            if i % 4 == 3:  # where the block's leading 1-byte codes make dp4a groups
                out |= {docs[i] - 1, docs[i], docs[i] + 1}
    if dense:
        out |= {(B.first >> DENSE_ALIGN) << DENSE_ALIGN, (((B.last[-1] >> DENSE_ALIGN) + 1) << DENSE_ALIGN) - 1}
    else:
        _, tf_shift, _ = tb.directory_lookup(G, index, term, np.zeros(0, np.uint32))
        if tf_shift < 32:
            s = 1 << tf_shift
            out |= set(range((B.first // s + 1) * s, B.last[-1] + 1, s))
    return np.array(sorted(x for x in out if 1 <= x <= TOP), np.uint32)


# ---------------------------------------------------------------------------------------------------------------- evaluation


def eval_sets(nodes, lists):
    """the docIDs node 0 matches, as a sorted uint32 array; lists[t] = the term's sorted docIDs.  Same semantics as pyeval.evaluate
    (AND / OR / NOT / MatchSome / Optional, and the reference's root-filter quirk), over sets instead of an ndocs + 1 mask"""
    empty = np.zeros(0, np.uint32)

    def term_docs(t):
        return empty if t == tb.EMPTY_TERM or t not in lists else np.asarray(lists[t], np.uint32)

    def rec(i):
        n = nodes[i]
        kind = int(n["kind"])
        if kind == tb.NODE_TERM:
            return term_docs(int(n["term"]))
        kids = [rec(int(n["first_child"]) + c) for c in range(int(n["nchildren"]))]
        if kind == tb.NODE_AND:
            out = kids[0]
            for k in kids[1:]:
                out = np.intersect1d(out, k, assume_unique=True)
            return out
        if kind == tb.NODE_OR:
            return np.unique(np.concatenate(kids)) if kids else empty
        if kind == tb.NODE_NOT:
            return np.setdiff1d(kids[0], kids[1], assume_unique=True)
        if kind == tb.NODE_SOME:
            u, cnt = np.unique(np.concatenate(kids), return_counts=True)
            return u[cnt >= int(n["term"])].astype(np.uint32)
        if kind == tb.NODE_OPTIONAL:
            return kids[0]
        raise ValueError(f"node kind {kind}")

    def cost(i):
        n = nodes[i]
        kind = int(n["kind"])
        if kind == tb.NODE_TERM:
            return len(term_docs(int(n["term"])))
        kids = [cost(int(n["first_child"]) + c) for c in range(int(n["nchildren"]))]
        if kind == tb.NODE_PHRASE:
            return min(kids)
        if kind in (tb.NODE_NOT, tb.NODE_OPTIONAL):
            return kids[0]
        if kind == tb.NODE_SOME:
            return sum(sorted(kids)[:max(0, len(kids) - int(n["term"]) + 1)])
        return min(kids) if kind == tb.NODE_AND else sum(kids)

    root, traversed = 0, False
    while int(nodes[root]["kind"]) == tb.NODE_NOT and cost(int(nodes[root]["first_child"]) + 1) <= cost(int(nodes[root]["first_child"])):
        root, traversed = int(nodes[root]["first_child"]), True
    if not (traversed and int(nodes[root]["kind"]) == tb.NODE_OR):
        root = 0
    return rec(root).astype(np.uint32)


def nblocks(terms, t):
    return (int(terms[t]["documents"]) + 31) // 32


def probe_order(nodes, terms):
    """(term ids in the planner's probe order, number of necessary terms, table over probe-order assignments) of a candidate plan: the
    necessary terms rarest first (the first one leads), then the others rarest first (plan_batch sorts by block count)"""
    tv, table, nec = tb.query_truth_table(nodes)
    n = len(tv)
    need = [j for j in range(n) if (nec >> j) & 1]
    rest = [j for j in range(n) if not (nec >> j) & 1]
    key = lambda j: nblocks(terms, tv[j])
    order = sorted(need, key=key) + sorted(rest, key=key)
    ptable = np.zeros(1 << n, bool)
    for pb in range(1 << n):
        bits = sum(1 << order[j] for j in range(n) if (pb >> j) & 1)
        ptable[pb] = table[bits]
    return [tv[j] for j in order], len(need), ptable


# ---------------------------------------------------------------------------------------------------------------- corpora


def _gaps(rng, kind, n):
    """n docID gaps of one block (the first is the gap from the previous block's last docID; the last one is carried by the block
    header, not by a code)"""
    one = lambda k: rng.integers(2, 128, k)
    two = lambda k: rng.integers(128, 1 << 14, k)
    three = lambda k: rng.integers(1 << 14, 40_000, k)
    g = one(n)
    if kind == "b2":
        g = two(n)
    elif kind == "mix12":
        g = np.where(rng.random(n) < 0.5, one(n), two(n))
    elif kind == "run3":  # a 2-byte codes, then 3-byte codes: the in-slot decode ends at (or just past) slot byte 80 for some a
        a = min(n, int(rng.integers(0, 30)))
        g = np.concatenate([two(a), three(n - a)])[:n]
    elif kind.startswith("c4") or kind.startswith("c5"):
        big = lambda: int(rng.integers(1 << 21, (1 << 21) + (1 << 20))) if kind[1] == "4" else int(rng.integers(1 << 28, (1 << 28) + 4096))
        at = {"first": 0, "mid": max(0, min(n - 2, int(rng.integers(1, 30)))), "last": max(0, n - 2)}[kind[2:]]
        g = np.where(rng.random(n) < 0.7, one(n), two(n))
        g[at] = big()
    return np.asarray(g, np.uint64)


LEAD_KINDS = ["b1", "b2", "mix12", "run3", "c4first", "b1", "run3", "c4mid", "mix12", "run3", "c4last", "b1"]


def lead_docs(rng, start, nblocks_, last_n, kinds, five=()):
    """docIDs of a lead of nblocks_ blocks (the last one of last_n documents), block b of kind kinds[b % len(kinds)], blocks listed
    in `five` of kind five[b] (5-byte codes)"""
    gaps = []
    for b in range(nblocks_):
        n = 32 if b + 1 < nblocks_ else last_n
        gaps.append(_gaps(rng, dict(five).get(b, kinds[b % len(kinds)]), n))
    d = np.uint64(start) + np.cumsum(np.concatenate(gaps))
    assert d[-1] <= TOP
    return d


def _u(*a):
    return np.unique(np.concatenate([np.asarray(x, np.uint64) for x in a])).astype(np.uint32)


# section A: leads of 1, 1, 31, 32, 33, 64 and 65 blocks (last blocks of 1, 2, 31, 32, 1, 31, 2 documents) whose blocks take every
# form of google_block_to_array; each with H (holds every lead document) and E (holds every other one), both with more blocks
LEADS = [("a1", 1, 1, ()), ("a2", 1, 2, ()), ("a31", 31, 31, ()), ("a32", 32, 32, ()),
         ("a33", 33, 1, ((3, "c5first"), (17, "c5mid"), (29, "c5last"))), ("a64", 64, 31, ()),
         ("a65", 65, 2, ((5, "c5mid"), (40, "c5first"), (63, "c5last")))]
DENSE_SPAN = 1 << 23


def lead_corpus(seed=7):
    """{name: docIDs} in index order: for every lead L of LEADS: L, Lh, Le; then "dense" (a resident bitmap over [1, 2^23]) and
    "filler" (no lead is the last term of the index: a mis-decoded lead block may read on past its term)"""
    rng = np.random.default_rng(seed)
    out = {}
    start = 1
    for k, (name, nb, last_n, five) in enumerate(LEADS):
        kinds = LEAD_KINDS[k % 3:] + LEAD_KINDS[: k % 3]
        L = lead_docs(rng, start + k, nb, last_n, kinds, five)
        extra = L[-1] + 2 + 3 * np.arange(40, dtype=np.uint64)
        out[name] = L.astype(np.uint32)
        out[name + "h"] = _u(L, L + 1, extra)
        out[name + "e"] = _u(L[::2], L + 1, extra)
    out["dense"] = np.arange(1, DENSE_SPAN, 3, dtype=np.uint32)
    out["filler"] = np.array([5, 9], np.uint32)
    return out


def probe_corpus(seed=3):
    """section B: probe terms "pn" (8 blocks: no table), "pt" (48 blocks: a table), "pb" (a resident bitmap, span ends not 2^17-
    aligned), the candidate sets qpn / qpt / qpb (probe_targets of each), a one-document term "zz" in none of them, and a filler"""
    rng = np.random.default_rng(seed)
    out = {}
    out["pn"] = lead_docs(rng, 1000, 8, 32, ["b1", "mix12", "c4mid", "run3", "b2", "b1", "c4last", "b1"]).astype(np.uint32)
    out["pt"] = lead_docs(rng, 3, 48, 32, ["b1", "b1", "mix12", "run3", "b2", "c4mid", "b1", "c4first"]).astype(np.uint32)
    d = np.arange(200_001, 700_001, dtype=np.uint32)
    out["pb"] = d[rng.random(len(d)) < 0.5]
    i, t, names = build({**out, "filler": np.array([1], np.uint32)})
    for name in ("pn", "pt", "pb"):
        out["q" + name] = probe_targets(i, term_tuple(t, names.index(name)), dense=name == "pb")
    out["zz"] = np.array([50_000_001], np.uint32)
    out["filler"] = np.array([3, 6], np.uint32)
    return out


def group_corpus(seed=5):
    """section D: lead "g" (161 blocks: five whole groups of 32 blocks and one of a single block; odd docIDs), "gp" (dense: every even
    docID and the documents of g's groups 0, 2, 4 and 5 — so groups 1 and 3 die at the first probe and group 0 survives whole), "godd"
    (dense: every odd docID — holds all of g), dense "d1" / "d2", "gx" / "gy" without a bitmap (the decoded operands of flat ANDs), and a
    filler"""
    rng = np.random.default_rng(seed)
    S = 400_000
    g = np.cumsum(rng.integers(1, 40, 161 * 32) * 2).astype(np.uint64) + 1
    g = g[: 160 * 32 + 1].astype(np.uint32)
    grp = np.arange(len(g)) // 1024
    out = {"g": g}
    out["gp"] = _u(np.arange(2, S + 1, 2), g[np.isin(grp, [0, 2, 4, 5])])
    out["godd"] = np.arange(1, S + 1, 2, dtype=np.uint32)
    out["d1"] = np.arange(3, S + 1, 3, dtype=np.uint32)
    out["d2"] = np.arange(5, S + 1, 5, dtype=np.uint32)
    out["gx"] = np.arange(11, S + 1, 43, dtype=np.uint32)
    out["gy"] = np.arange(17, S + 1, 53, dtype=np.uint32)
    out["filler"] = np.array([4, 8], np.uint32)
    return out


def truth_corpus(ns=range(2, 9), seed=9):
    """section C: for every n, terms x{n}t0 .. x{n}t{n-1}: one document per assignment of the n terms (document base + r * 2^n + a holds
    exactly the terms whose bit is set in a), replicated until every term has more than 64 blocks, plus documents that hold a single
    term, more of them for the earlier terms of the tree — so the probe order (rarest first) is not the tree order"""
    rng = np.random.default_rng(seed)
    out = {}
    base = 1
    for n in ns:
        reps = (64 * 32 * 2) // (1 << (n - 1)) + 2
        a = np.arange(1 << n)
        docs = base + (np.arange(reps)[:, None] * (1 << n) + a[None, :]).ravel()
        held = np.tile(a, reps)
        top = int(docs[-1]) + 1
        for j in range(n):
            extra = top + np.sort(rng.choice(20_000, size=(n - j) * 900, replace=False)) * n + j
            out[f"x{n}t{j}"] = _u(docs[(held >> j) & 1 == 1], extra)
        base = int(max(int(v[-1]) for k, v in out.items() if k.startswith(f"x{n}t"))) + 100
    out["filler"] = np.array([base + 10], np.uint32)
    return out


def top_corpus(seed=13):
    """section F: docIDs that end at 2^32 - 2: a lead "fl" with 5-byte codes as first, middle and last delta of its blocks and
    2^32 - 2 as its last docID, "fp" (holds every lead document, 5-byte codes mid-block, ends at 2^32 - 2), "fb" (a resident bitmap
    ending at 2^32 - 2), the candidate sets of fp's and fb's switch points (qfp, qfb), and a filler"""
    rng = np.random.default_rng(seed)
    L = lead_docs(rng, 0, 40, 32, ["b1", "mix12", "c4mid", "b2", "run3"], five=((2, "c5mid"), (9, "c5first"), (20, "c5last")))
    L = L + np.uint64(TOP) - L[-1]
    out = {"fl": L.astype(np.uint32)}
    P = lead_docs(rng, 0, 30, 32, ["b1", "b1", "c4first", "mix12"], five=((4, "c5mid"), (12, "c5mid")))
    P = P + np.uint64(TOP) - P[-1]
    out["fp"] = _u(L, P)
    d = np.arange(TOP - 400_000, TOP + 1, dtype=np.uint64)
    out["fb"] = _u(d[rng.random(len(d)) < 0.4], [TOP])
    i, t, names = build({**out, "filler": np.array([1], np.uint32)})
    for name in ("fp", "fb"):
        out["q" + name] = probe_targets(i, term_tuple(t, names.index(name)), dense=name == "fb")
    out["zz"] = np.array([7], np.uint32)
    out["filler"] = np.array([3, 6], np.uint32)
    return out


def build(lists, names=None):
    """(index, terms, names) of a GOOGLE index with one term per list, in order"""
    names = list(names or lists)
    b = tb.IndexBuilder(G)
    for n in names:
        d = np.asarray(lists[n], np.uint32)
        b.add_term(d, 1 + (d % 3).astype(np.uint32))
    return b.index(), b.terms_array(), names


# ---------------------------------------------------------------------------------------------------------------- queries
# (text, parser flags, min_match): flags 8 = <expr> is Optional, 16 = [a, b, ...] is MatchSome (refharness.RefIndex.exec)


def lead_queries():
    """section A: every lead against the term that holds all its documents and the one that holds every other one"""
    return [(f"{L} AND {L}{s}", 0, 0) for L, *_ in LEADS for s in ("h", "e")]


def mixed_lead_queries():
    """section A on the mixed-run tickets: every lead as the decoded operand of a flat AND with a bitmap operand"""
    return [(f"{L} AND dense", 0, 0) for L, *_ in LEADS]


PROBE_QUERIES = [(f"q{p} AND ({p} OR zz)", 0, 0) for p in ("pn", "pt", "pb")] + [(f"q{p} AND {p}", 0, 0) for p in ("pn", "pt", "pb")]
TOP_QUERIES = [("fl AND fp", 0, 0), ("fl AND fb", 0, 0), ("fl AND (fp OR fb)", 0, 0), ("qfp AND (fp OR zz)", 0, 0),
               ("qfb AND (fb OR zz)", 0, 0), ("qfp AND fp", 0, 0), ("qfb AND fb AND fp", 0, 0)]


def truth_queries(n):
    """section C over x{n}t0 .. x{n}t{n-1}: AND, AND / OR, AND / OR / NOT, MatchSome at min 1, m - 1 and m, Optional, each with 1 ..
    n - 1 necessary terms"""
    a = [f"x{n}t{j}" for j in range(n)]
    qs = [(" AND ".join(a), 0, 0)]
    for k in range(1, n):
        nec, rest = " AND ".join(a[:k]), a[k:]
        qs.append((f"{nec} AND ({' OR '.join(rest)})", 0, 0))
        if len(rest) >= 2:
            qs.append((f"{nec} AND ({' OR '.join(rest[:-1])}) NOT {rest[-1]}", 0, 0))
        qs.append((f"{nec} " + " ".join(f"<{x}>" for x in rest), 8, 0))
        if len(rest) >= 2:
            for m in sorted({1, len(rest) - 1, len(rest)}):
                qs.append((f"{nec} AND [{', '.join(rest)}]", 16, m))
    if n >= 4:
        qs.append((f"{a[0]} AND (({a[1]} AND {a[2]}) OR ({' OR '.join(a[3:])} NOT {a[1]}))", 0, 0))
    return qs


# n = 8: queries whose matches lie in every word of the 256-bit table (probe position 7 present and absent), and miss in every word
WIDE_QUERIES = [("x8t0 AND [x8t1, x8t2, x8t3, x8t4, x8t5, x8t6, x8t7]", 16, 4),
                ("x8t0 AND ((x8t1 OR x8t2 OR x8t3 OR x8t4) NOT (x8t5 AND x8t6)) AND (x8t7 OR x8t2 OR x8t4)", 0, 0)]


def all_truth_queries():
    return [q for n in range(2, 9) for q in truth_queries(n)] + WIDE_QUERIES


# section D: one batch of every route of the DocumentsOnly launch around the candidate-driven queries (default crossover)
GROUP_ROUTES = {
    "g AND gp": tb.ROUTE_CANDIDATE,  # groups 1 and 3 die at the first probe, group 0 survives whole
    "g AND godd": tb.ROUTE_CANDIDATE,  # every candidate survives: the result is its segment bound
    "g AND (gp OR d1)": tb.ROUTE_CANDIDATE,  # membership bytes
    "gx AND d1": tb.ROUTE_FLAT_AND,  # one decoded operand: mixed-run tickets
    "d1 AND d2": tb.ROUTE_FLAT_AND,  # all-bitmap
    "gx AND gy": tb.ROUTE_FLAT_AND,  # two decoded operands
    "(gx OR gy) AND d1 NOT d2": tb.ROUTE_FLAT_TREE,
}
# section E: the candidate queries without and with membership bytes, and flat ANDs with one decoded operand
CAND_PLAIN = ["g AND gp", "g AND godd"]
CAND_MEMBER = ["g AND (gp OR d1)"]
FLAT_MIXED = ["gx AND d1", "gy AND d2"]


def parse(queries, tdict):
    return [tb.parse_query(q, tdict, min_match=m or None) for q, _, m in queries]


def own_slots(index, terms, plans):
    """the docset slots the batch's step programs need (the planner's own minimum)"""
    return max(tb.debug_compile(G, index, terms, p, False)[2] for p in plans)


def cand_smem_slots(docs_shift, membership, own=0):
    """the docset slots a batch with a candidate query gets at this tile size (planner.cpp: the candidate array, one gather buffer and,
    with membership bytes, one byte per candidate must fit the warp's share: slots x 2^shift / 8 bytes + the staging area)"""
    stage = 32 * GATHER + 512
    need = 33 * 32 * 4 + 32 * GATHER + (33 * 32 if membership else 0)
    slot = (1 << docs_shift) // 8
    return max(own, -(-(need - stage) // slot))
