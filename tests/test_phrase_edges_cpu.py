"""Phrases of up to 16 terms — the corpus, the queries and the CPU pins that tests/test_gpu_phrase_edges.py runs on the device.

The corpus is built document by document, one term per position (the reference's DocWordsSpace keeps one term per position), every
position given explicitly, so that the answer of every query is known by construction:
  * a 16-token sentence S whose terms repeat on both sides of each OP_ARG boundary (j = 3/4, 7/8, 11/12) and whose ids are large and
    differ in both low bytes — except s6, which is term id 0, the value of an OP_ARG padding word;
  * S at the start of a document, in its middle and ending at position 16 383 (the last legal one); each k-prefix followed by a wrong
    token; S with one token replaced, and S with a one-position gap before one token, for every j;
  * S twice or three times 63, 64, 8 191 and 8 192 positions apart (GOOGLE hit steps `delta << 1 | flag` of 1 / 2 and 2 / 3 bytes);
  * runs of s0 whose position deltas are mostly small with a few larger (PFor exceptions of width 1) or very large ones (width > 1);
  * S 300 times, 17 positions apart, in the last document: more than 64 starts of t0, constant deltas of the once-per-sentence terms
    (LUCENE hit pages with L == 0), and every sentence term's last document running from its full 128-hit blocks into the varbyte tail;
  * two sentences P and Q of 16 distinct terms each, no term shared with S or with each other (32 distinct terms: the collect pass's limit);
  * terms f1 .. f5 for the trees and dense terms d2, d3, d5 (resident GOOGLE bitmaps) over every document.
Pinned here: pyeval.evaluate gives the planted answer for every query, the planner packs each k-term phrase into
ceil(k / 4) OP_ARG steps that phrase_arg reads back in order (also behind OP_SLOT AND in the deferred scoring pass), the kernels' position
cursors (trn_debug_positions) read the sentence terms exactly, the routes, the collect pass's 32-term limit, the refusal of phrases of
1 and 17 terms, and the percolator's anchors."""
import numpy as np
import pytest

import trinity_b200 as tb
from matchutil import host_build, payload_hits
from percutil import RefPercolator, evaluate as perc_evaluate
from pyeval import evaluate
from stepsim import M_AND, OP_SLOT
from trinity_b200._ffi import QNODE_DTYPE

OP_PHRASE, OP_ARG = 7, 8
NDOCS = 300_000
STRIDE = 3119  # planted documents: docIDs 7, 7 + STRIDE, ... (spread over the tiles of every TRN_DOCS_SHIFT)
MAX_POS = 16383  # the last legal position (Limits::MaxPosition = 16384)
FREE = 16300  # positions 16300 .. 16312 carry f1 .. f5 and d2, d3, d5; no planted token reaches them (the end document starts at 16368)

# ------------------------------------------------------------------------------------------------ the vocabulary
V = 0x13000  # 77 824 terms: most hold no document
_big = lambda k: 0x10000 + 0x111 * k  # k = 1 .. 11: ids above 2^16 that differ from each other in both low bytes
a, b, c, d, e, f, g, h, i, j, k = (_big(x) for x in range(1, 12))
Z = 0  # term id 0: what an OP_ARG padding word holds
S = [a, b, c, d, d, e, Z, f, f, g, a, h, h, i, j, k]
P = [0x11000 + 0x0F1 * x for x in range(16)]
Q = [0x12000 + 0x0E3 * x for x in range(16)]
W, X = 1, 2  # the wrong token of near misses and prefixes; filler
F = [3, 4, 5, 6, 7]  # f1 .. f5
DENSE = {"d2": (8, 2), "d3": (9, 3), "d5": (10, 5)}  # name: (term id, every n-th document)
NAMES = [f"v{x}" for x in range(V)]
NAMES[W], NAMES[X] = "w", "x"
for n_, t_ in zip(("f1", "f2", "f3", "f4", "f5"), F):
    NAMES[t_] = n_
for n_, (t_, _) in DENSE.items():
    NAMES[t_] = n_
assert len(set(S) | set(P) | set(Q) | {W, X, *F, 8, 9, 10}) == 11 + 1 + 32 + 10
assert S[3] == S[4] and S[7] == S[8] and S[11] == S[12] and S[6] == 0


def text(terms):
    return '"' + " ".join("nosuch" if t is None else NAMES[t] for t in terms) + '"'


# ------------------------------------------------------------------------------------------------ the planted documents
def _doc(*parts):
    """{position: term} from (start position, tokens) parts; one term per position"""
    out = {}
    for start, toks in parts:
        for n_, t_ in enumerate(toks):
            assert start + n_ not in out and 1 <= start + n_ < FREE or start + n_ > FREE + 12, (start, n_)
            assert start + n_ <= MAX_POS
            out[start + n_] = t_
    return out


def _run(rng, n, small, big, nbig):
    """n positions of one term: deltas drawn from `small`, `nbig` of them from `big` (PFor exceptions in the LUCENE hit pages)"""
    dl = rng.choice(small, n)
    dl[rng.choice(np.arange(1, n), nbig, replace=False)] = rng.choice(big, nbig)
    return np.cumsum(dl)


def _planted():
    rng = np.random.default_rng(16)
    docs = [("start", _doc((1, S))), ("middle", _doc((4000, [X]), (5000, S), (5017, [X]))), ("end", _doc((1, [X]), (MAX_POS - 15, S)))]
    docs += [(f"prefix{n_}", _doc((1, S[:n_] + [W]))) for n_ in range(2, 17)]
    docs += [(f"miss{x}", _doc((1, S[:x] + [W] + S[x + 1:]))) for x in range(16)]
    docs += [(f"gap{x}", _doc((1, S[:x]), (2 + x, S[x:]))) for x in range(1, 16)]
    for dl in (63, 64, 8191, 8192):
        docs.append((f"spaced{dl}", _doc(*[(1 + r * dl, S) for r in range(3 if dl < 100 else 2)])))
    for name, small, big, nbig in (("run-k1", [1, 2, 3], [5, 6, 7], 3), ("run-kbig", [1, 2], [700, 1500, 2600], 3)):
        pos = _run(rng, 400, small, big, nbig)
        docs.append((name, _doc(*[(int(p), [a]) for p in pos], (int(pos[-1]) + 5, S))))
    docs += [("P", _doc((1, P))), ("Q", _doc((3, Q))), ("PQ", _doc((1, P), (40, Q))), ("QP", _doc((1, Q), (17, P))),
             ("Pmiss7", _doc((1, P[:7] + [W] + P[8:]), (30, Q))), ("SP", _doc((1, S), (20, P[:9]), (33, [X])))]
    docs.append(("many", _doc(*[(1 + 17 * r, S + [X]) for r in range(300)])))  # last: the sentence terms' last document
    return docs


PLANTED = _planted()
DOCIDS = [7 + STRIDE * n_ for n_ in range(len(PLANTED))]
TAG = {tag: did for (tag, _), did in zip(PLANTED, DOCIDS)}
assert DOCIDS[-1] <= NDOCS


def _f_docs(n_):
    """docIDs of f(n_+1): planted documents by index pattern and every (11 + 2 n_)-th document"""
    pat = [lambda x: x % 2 == 0, lambda x: x % 3 == 0, lambda x: x % 2 == 1 or x % 5 == 0, lambda x: x % 7 == 0, lambda x: x % 3 == 1][n_]
    return np.union1d([DOCIDS[x] for x in range(len(PLANTED)) if pat(x)], np.arange(11 + 2 * n_, NDOCS + 1, 11 + 2 * n_)).astype(np.uint32)


def _postings():
    """term id -> (docids, freqs, positions) for every term that holds a document"""
    per = {}
    for did, (_, doc) in zip(DOCIDS, PLANTED):
        for p_, t_ in sorted(doc.items()):
            per.setdefault(t_, {}).setdefault(did, []).append(p_)
    out = {}
    for t_, m in per.items():
        ds = np.array(sorted(m), np.uint32)
        out[t_] = (ds, np.array([len(m[int(x)]) for x in ds], np.uint32), np.array([p_ for x in ds for p_ in m[int(x)]], np.uint32))
    for n_, t_ in enumerate(F):
        ds = _f_docs(n_)
        out[t_] = (ds, np.ones(len(ds), np.uint32), np.full(len(ds), FREE + n_, np.uint32))
    for n_, (t_, every) in enumerate(DENSE.values()):
        ds = np.arange(every, NDOCS + 1, every, dtype=np.uint32)
        out[t_] = (ds, np.ones(len(ds), np.uint32), np.full(len(ds), FREE + 10 + n_, np.uint32))
    return out


POSTINGS = _postings()
EMPTY = np.zeros(0, np.uint32)


def lists(shift=0):
    """[(docids, freqs, positions)] of every term id, docIDs moved up by `shift`"""
    out = []
    for t_ in range(V):
        ds, fs, ps = POSTINGS.get(t_, (EMPTY, EMPTY, EMPTY))
        out.append(((ds.astype(np.uint64) + shift).astype(np.uint32), fs, ps))
    return out


def payload_lists():
    """the same postings with payloads: sizes 0..8 that change inside a document (matchutil.payload_hits)"""
    rng = np.random.default_rng(8)
    return [(ds, fs, ps, *payload_hits(rng, len(ps))) for ds, fs, ps in lists()]


def build(codec, ls=None):
    """(index, hits, terms) through the host IndexBuilder"""
    bld = tb.IndexBuilder(codec)
    for ds, fs, ps in ls if ls is not None else lists():
        bld.add_term(ds, fs, ps)
    return bld.index(), bld.hits(), bld.terms_array()


# ------------------------------------------------------------------------------------------------ the answers by construction
def planted_phrase(terms):
    """docIDs of the planted documents that hold the phrase (a non-zero position p with terms[j] at p + j for every j)"""
    if None in terms:
        return set()
    return {did for did, (_, doc) in zip(DOCIDS, PLANTED) if any(all(doc.get(p_ + o) == t_ for o, t_ in enumerate(terms)) for p_ in doc)}


def _starts(fs):
    """hit number where each document's hits start, and the total"""
    return np.concatenate([[0], np.cumsum(fs.astype(np.int64))])


def holds(t_):
    return set(POSTINGS[t_][0].tolist())


def _queries():
    """[(text, planted answer)]: every phrase and tree the device is checked on"""
    qs = [(text(S[:n_]), planted_phrase(S[:n_])) for n_ in range(2, 17)]
    qs += [(text(S[x:y]), planted_phrase(S[x:y])) for x, y in ((3, 11), (6, 14), (8, 16), (1, 16), (12, 16))]
    for x in (5, 9, 15):  # an unknown term: OP_CLEAR
        qs.append((text(S[:x] + [None] + S[x + 1:]), set()))
    qs += [(text(S + [W]), planted_phrase(S)), (text(S + [W, X, W, a]), planted_phrase(S))]  # the parser keeps 16 terms, as the reference
    qs += [(text(P), planted_phrase(P)), (text(Q), planted_phrase(Q)), (text(P[:9]), planted_phrase(P[:9]))]
    f1, f2, f3, f4, f5 = (holds(t_) for t_ in F)
    qs += [(text(S) + " AND f1", planted_phrase(S) & f1),
           ("f1 NOT " + text(S[:8]), f1 - planted_phrase(S[:8])),
           (f"(f2 OR {text(S[:5])}) AND f3", (f2 | planted_phrase(S[:5])) & f3),  # deferred scoring pass, one condition
           (f"f3 AND (f4 OR ({text(S[3:9])} AND (f5 OR {text(P[:9])})))",  # nested conditions: OP_SLOT AND mask before OP_PHRASE
            f3 & (f4 | (planted_phrase(S[3:9]) & (f5 | planted_phrase(P[:9]))))),
           (text(P) + " AND " + text(Q), planted_phrase(P) & planted_phrase(Q))]  # 32 distinct terms
    return qs


QUERIES = _queries()
TEXTS = [q for q, _ in QUERIES]
WANT = [np.array(sorted(w), np.uint32) for _, w in QUERIES]
TD = None


def tdict():
    global TD
    if TD is None:
        TD = tb.TermDictionary(NAMES)
    return TD


# the non-phrase plans of the mixed batch: all-bitmap, flat AND, flat OR, flat tree
OTHERS = ["d2 AND d3", "d3 AND d5 AND d2", "f1 AND f2", "f1 AND d2", "f1 OR f2 OR f3", "(f1 OR d5) AND (f2 OR d3) NOT f4"]


def hand_phrase(n_):
    """a phrase node of n_ children built by hand (the parser would make one term of 1 and cut 17 down to 16)"""
    arr = np.zeros(1 + n_, QNODE_DTYPE)
    arr[0] = (tb.NODE_PHRASE, n_, 1, 0, 0.0)
    for x in range(n_):
        arr[1 + x] = (tb.NODE_TERM, 0, 0, S[x % 16], 0.0)
    return arr


# ------------------------------------------------------------------------------------------------ CPU pins
def test_the_planted_documents_make_every_case():
    """each near miss and gap is really rejected, each prefix matches, and the layout edges are in the corpus"""
    ph = planted_phrase(S)
    assert {TAG["start"], TAG["middle"], TAG["end"], TAG["many"], TAG["prefix16"], TAG["run-k1"], TAG["run-kbig"], TAG["SP"]} <= ph
    assert max(PLANTED[DOCIDS.index(TAG["end"])][1]) == MAX_POS
    for x in range(16):
        assert TAG[f"miss{x}"] not in ph
    for x in range(1, 16):
        assert TAG[f"gap{x}"] not in ph
        assert x < 2 or TAG[f"gap{x}"] in planted_phrase(S[:x])
        assert x > 14 or TAG[f"gap{x}"] in planted_phrase(S[x:])
    for n_ in range(2, 17):
        assert TAG[f"prefix{n_}"] in planted_phrase(S[:n_])
        assert n_ == 16 or TAG[f"prefix{n_}"] not in planted_phrase(S[:n_ + 1])
    assert TAG["Pmiss7"] not in planted_phrase(P) and TAG["Pmiss7"] in planted_phrase(Q)
    assert planted_phrase(S + [W]) == {TAG["prefix16"]} != planted_phrase(S)  # so the 17-term query shows the truncation
    assert all(len(w) for q, w in zip(TEXTS, WANT) if "nosuch" not in q)
    assert sum(1 for p_ in PLANTED[-1][1] if PLANTED[-1][1][p_] == a and PLANTED[-1][1].get(p_ + 1) == b) == 300  # > 64 starts of t0
    # GOOGLE hit steps of 1, 2 and 3 bytes: consecutive hits of a sentence term 63, 64, 8191 and 8192 positions apart
    deltas = set()
    for t_ in S:
        ds, fs, ps = POSTINGS[t_]
        at = _starts(fs)
        for x in range(len(ds)):
            deltas |= set(np.diff(ps[at[x]:at[x + 1]]).tolist())
    assert {63, 64, 8191, 8192} <= deltas


def _lucene_deltas(t_):
    """the LUCENE hit stream of a term: position deltas (restarting from 0 in every document), and the hit number where each document starts"""
    ds, fs, ps = POSTINGS[t_]
    at = _starts(fs).astype(np.int64)
    dl = ps.astype(np.int64).copy()
    for x in range(len(ds)):
        dl[at[x] + 1:at[x + 1]] = np.diff(ps[at[x]:at[x + 1]])
    return dl, at


def test_the_lucene_hit_pages_take_every_form():
    """L == 0 pages (128 equal deltas), pages with exceptions, and a last document whose hits run from a full block into the tail"""
    for t_ in set(S):
        dl, at = _lucene_deltas(t_)
        pages = dl[: len(dl) // 128 * 128].reshape(-1, 128)
        assert S.count(t_) > 1 or np.any(pages.max(1) == pages.min(1)), t_  # the once-per-sentence terms: an L == 0 page
        assert len(dl) % 128 and at[-2] < len(dl) // 128 * 128, t_  # the last document crosses into the tail
    dl, _ = _lucene_deltas(a)
    pages = dl[: len(dl) // 128 * 128].reshape(-1, 128)
    small = pages[(np.sort(pages, 1)[:, -4] <= 3)]
    assert any(p_.max() in (5, 6, 7) for p_ in small) and any(p_.max() >= 700 for p_ in small)  # exception widths 1 and > 1


def restated(q):
    """pyeval.evaluate of query q with BM25 weights: (match mask, scores) over docIDs 0 .. NDOCS"""
    nodes = tb.parse_query(q, tdict())
    for x in nodes:
        if x["kind"] == tb.NODE_TERM and x["term"] != tb.EMPTY_TERM:
            x["weight"] = tb.bm25_idf(len(POSTINGS.get(int(x["term"]), (EMPTY,))[0]), NDOCS)
    return evaluate(nodes, _PL, NDOCS, weights=True, positions=_POS)


def _restated_inputs():
    pl = [POSTINGS.get(t_, (EMPTY, EMPTY))[:2] for t_ in range(V)]
    pos = [{}] * V
    for t_ in set(S) | set(P) | set(Q):
        ds, fs, ps = POSTINGS[t_]
        at = _starts(fs)
        pos[t_] = {int(x): ps[at[n_]:at[n_ + 1]].tolist() for n_, x in enumerate(ds)}
    return pl, pos


_PL, _POS = _restated_inputs()


def test_pyeval_gives_the_planted_answers():
    """pyeval.evaluate (the structural restatement pinned against the reference's exec_query in test_phrase_cpu) agrees with the
    construction.  The device is checked against these answers: the reference's exec_query was not stable on this corpus (heap
    corruption: intermittent aborts and a wrong answer now and then, in its DocumentsOnly, scored and default exec modes alike)."""
    for q, want in zip(TEXTS, WANT):
        m, _ = restated(q)
        assert np.array_equal(np.flatnonzero(m), want), q


def _phrase_args(steps, at):
    """the term ids OP_PHRASE step `at` names, read by phrase_arg's rule: per OP_ARG step term, pad2, idf low word, idf high word"""
    k_ = int(steps[at]["mode"])
    n_ = (k_ + 3) // 4
    args = steps[at + 1: at + 1 + n_]
    assert len(args) == n_ and all(int(s_["op"]) == OP_ARG for s_ in args), (k_, steps["op"][at:at + n_ + 2])
    assert at + 1 + n_ == len(steps) or int(steps[at + 1 + n_]["op"]) != OP_ARG  # exactly ceil(k / 4) of them
    words = []
    for s_ in args:
        idf = int(np.array([s_["idf"]], np.float64).view(np.uint64)[0])
        words += [int(s_["term"]), int(s_["pad2"]), idf & 0xFFFFFFFF, idf >> 32]
    assert words[k_:] == [0] * (len(words) - k_)  # padding
    return words[:k_]


@pytest.fixture(scope="module")
def google_index():
    index, _, terms = build(tb.CODEC_GOOGLE)
    return index, terms


@pytest.mark.parametrize("scored", [False, True], ids=["docs", "scored"])
def test_every_phrase_packs_its_term_ids_into_op_arg_steps(google_index, scored):
    index, terms = google_index
    seen = set()
    for ph in [S[:n_] for n_ in range(2, 17)] + [S[3:11], S[6:14], S[1:16], P, Q, P[:9]]:
        steps, _, _ = tb.debug_compile(tb.CODEC_GOOGLE, index, terms, tb.parse_query(text(ph), tdict()), scored)
        at = [n_ for n_, s_ in enumerate(steps) if int(s_["op"]) == OP_PHRASE]
        assert len(at) == 1 and int(steps[at[0]]["mode"]) == len(ph)
        assert _phrase_args(steps, at[0]) == ph, ph
        seen.add(len(ph))
    assert seen == set(range(2, 17))
    steps, _, _ = tb.debug_compile(tb.CODEC_GOOGLE, index, terms, tb.parse_query(text(S[:9] + [None] + S[10:]), tdict()), scored)
    assert OP_PHRASE not in steps["op"].tolist()  # an unknown term: OP_CLEAR


def test_the_deferred_pass_masks_the_phrase_and_keeps_its_args_together(google_index):
    index, terms = google_index
    for q, ph, nested in ((TEXTS[-2], P[:9], True), (TEXTS[-2], S[3:9], False)):
        steps, _, _ = tb.debug_compile(tb.CODEC_GOOGLE, index, terms, tb.parse_query(q, tdict()), True)
        at = [n_ for n_, s_ in enumerate(steps) if int(s_["op"]) == OP_PHRASE and int(s_["mode"]) == len(ph) and _phrase_args(steps, n_) == ph]
        assert at, (q, ph)  # (the last one: the check of the deferred scoring pass)
        last = at[-1]
        assert int(steps[last]["flags"]) & 1  # F_SCORE
        sl = steps[last - 1]
        assert int(sl["op"]) == OP_SLOT and int(sl["mode"]) == M_AND and int(sl["dst"]) == int(steps[last]["dst"]), steps[last - 1]
        mask = int(sl["src"])
        # with nested conditions the mask slot is built from several conditions (OP_SLOT SET, then AND) just before
        built = [s_ for s_ in steps[:last] if int(s_["op"]) == OP_SLOT and int(s_["dst"]) == mask]
        assert len(built) >= 2 or not nested, (q, ph, built)


@pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
@pytest.mark.parametrize("payloads", [False, True], ids=["plain", "payloads"])
def test_the_position_cursors_read_the_sentence_terms(codec, payloads):
    ls = payload_lists() if payloads else lists()
    index, hits, terms = host_build(codec, ls) if payloads else build(codec, ls)
    for t_ in sorted(set(S) | set(P)):
        ds, fs, ps = POSTINGS[t_]
        at = _starts(fs)
        got = tb.debug_positions(codec, index, hits, terms[t_], ds)
        for n_ in range(len(ds)):
            assert np.array_equal(got[n_], ps[at[n_]:at[n_ + 1]]), (codec, t_, int(ds[n_]))


def test_routes():
    """every query with a phrase runs the step program (DocumentsOnly) and k_exec_tiles (scored); a phrase in the batch keeps the
    non-phrase plans on their routes but takes them off the run-major tickets (planned for GOOGLE: a LUCENE plan with a phrase needs the
    hits.data of an uploaded source)"""
    index, _, terms = build(tb.CODEC_GOOGLE)
    plans = [tb.parse_query(q, tdict()) for q in TEXTS]
    for mode, route in ((tb.MODE_DOCS_ONLY, tb.ROUTE_STEPS), (tb.MODE_SCORED_ALL, tb.ROUTE_EXEC_TILES)):
        routes, _ = tb.debug_plan(tb.CODEC_GOOGLE, index, terms, plans, mode, max_docid=NDOCS)
        assert routes.tolist() == [route] * len(plans), (mode, routes)
    others = [tb.parse_query(q, tdict()) for q in OTHERS]
    alone, _ = tb.debug_plan(tb.CODEC_GOOGLE, index, terms, others, tb.MODE_DOCS_ONLY, max_docid=NDOCS)
    assert {tb.ROUTE_FLAT_AND, tb.ROUTE_FLAT_OR, tb.ROUTE_FLAT_TREE} <= set(alone.tolist()), alone
    off, _ = tb.debug_dense_terms(tb.CODEC_GOOGLE, index, terms)
    assert all(off[t_] != tb.DENSE_NONE for t_, _ in DENSE.values())
    assert len(tb.debug_dense_runs(tb.CODEC_GOOGLE, index, terms, others, tb.MODE_DOCS_ONLY, max_docid=NDOCS)[1])
    mixed = others + [tb.parse_query(text(S), tdict())]
    beside, _ = tb.debug_plan(tb.CODEC_GOOGLE, index, terms, mixed, tb.MODE_DOCS_ONLY, max_docid=NDOCS)
    assert beside.tolist()[:len(others)] == alone.tolist()
    assert len(tb.debug_dense_runs(tb.CODEC_GOOGLE, index, terms, mixed, tb.MODE_DOCS_ONLY, max_docid=NDOCS)[1]) == 0
    assert len(tb.debug_mixed_runs(tb.CODEC_GOOGLE, index, terms, mixed, tb.MODE_DOCS_ONLY, max_docid=NDOCS)[1]) == 0


def test_the_collect_pass_takes_32_distinct_terms_and_refuses_33(google_index):
    index, terms = google_index
    ok = tb.parse_query(TEXTS[-1], tdict())
    assert len({int(x["term"]) for x in ok if x["kind"] == tb.NODE_TERM}) == 32
    tb.debug_plan(tb.CODEC_GOOGLE, index, terms, [ok], tb.MODE_MATCHED_TERMS, max_docid=NDOCS)
    with pytest.raises(tb.TrinityError, match="32 distinct terms"):
        tb.debug_plan(tb.CODEC_GOOGLE, index, terms, [tb.parse_query(TEXTS[-1] + " AND f1", tdict())], tb.MODE_MATCHED_TERMS, max_docid=NDOCS)


@pytest.mark.parametrize("n", [1, 17])
def test_phrases_of_1_and_17_terms_are_refused(google_index, n):
    index, terms = google_index
    for mode in (tb.MODE_DOCS_ONLY, tb.MODE_SCORED_ALL, tb.MODE_MATCHED_TERMS):
        with pytest.raises(tb.TrinityError, match="2..16 terms"):
            tb.debug_plan(tb.CODEC_GOOGLE, index, terms, [hand_phrase(n)], mode, max_docid=NDOCS)
    with pytest.raises(tb.TrinityError, match="2..16 terms"):
        tb.debug_percolator_plan([hand_phrase(n)], V)


# ------------------------------------------------------------------------------------------------ the percolator's phrases
PERC_PHRASES = [S[:5], S[:9], S, P[:5], P[:9], P]


def perc_costs():
    """three cost arrays: the anchor (the first occurrence of the cheapest term) at index 0, in the middle and at k - 1 of the P phrases"""
    out = []
    for rank in (lambda x: x, lambda x: abs(x - 2), lambda x: 16 - x):
        cost = np.full(V, 100, np.uint32)
        for ph in (S, P):
            for x in range(16):
                if ph.index(ph[x]) == x:
                    cost[ph[x]] = 1 + rank(x)
        out.append(cost)
    return out


def perc_docs():
    """token arrays: every phrase alone (exactly as long), at token 0, ending at the last token, one token short, and a near miss at every j"""
    docs = []
    for ph in PERC_PHRASES:
        ph = list(ph)
        docs += [np.array(x, np.uint32) for x in (ph, ph + [X, X], [X, W] + ph, ph[:-1], ph[1:], [X] + ph[:-1])]
        for x in range(len(ph)):
            docs.append(np.array(ph[:x] + [W] + ph[x + 1:], np.uint32))
            docs.append(np.array([X] + ph[:x] + [tb.EMPTY_TERM] + ph[x + 1:], np.uint32))
    return docs


def test_percolator_anchors_and_meaning():
    plans = [tb.parse_query(text(ph), tdict()) for ph in PERC_PHRASES]
    anchors = {}
    for cost in perc_costs():
        for ph, (status, cov) in zip(PERC_PHRASES, tb.debug_percolator_plan(plans, V, term_cost=cost)):
            best = min(ph, key=lambda t_: (int(cost[t_]), t_))
            assert status == 0 and cov == [best]
            anchors.setdefault(len(ph) if ph[0] == P[0] else -len(ph), set()).add(ph.index(best))
    for n_ in (5, 9, 16):
        assert {0, n_ - 1} < anchors[n_] and len(anchors[n_]) == 3, anchors  # the P phrases: anchor 0, a middle one and k - 1
    docs = perc_docs()
    want = RefPercolator([(text(ph), 0, 0) for ph in PERC_PHRASES], vocab=NAMES).run(docs)
    for qi, nodes in enumerate(plans):
        got = [perc_evaluate(nodes, x) for x in docs]
        assert got == [qi in set(w.tolist()) for w in want], text(PERC_PHRASES[qi])
        assert sum(got) >= 3
