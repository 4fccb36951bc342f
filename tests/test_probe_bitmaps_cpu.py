"""The second tier of resident bitmaps, the probe bitmaps that only the candidate-driven conjunction reads (planner.h select_probe_terms),
checked without a GPU through trn_debug_probe_terms against a restatement in Python:
  * a GOOGLE term without a dense bitmap qualifies when its bitmap is at most TRN_PROBE_RATIO (16) times its chunk; qualifying terms are
    taken densest first (ties: lower term id) while the tier fits TRN_PROBE_BUDGET (2.0) x the index bytes and both tiers together
    fewer than 2^32 words; the tier is laid out behind the dense bitmaps, and a dense term keeps its dense offset;
  * TRN_PROBE_BITMAPS=0, TRN_PROBE_BUDGET=0, TRN_DENSE_BITMAPS=0 and LUCENE sources give none;
  * a term whose span ends at 2^32;
  * the planner does not see the tier: the dense selection, every route and every run ticket are the same with the tier on and off."""
import contextlib
import os

import numpy as np
import pytest

import bench
import candutil as cu
import trinity_b200 as tb

G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE
NONE = tb.DENSE_NONE
ALIGN = 1 << 17
TOP = 2**32 - 2
KNOBS = ("TRN_PROBE_BITMAPS", "TRN_PROBE_RATIO", "TRN_PROBE_BUDGET", "TRN_DENSE_BITMAPS", "TRN_DENSE_BUDGET", "TRN_CAND_COST")


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


@contextlib.contextmanager
def _env(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _span_words(first: int, last: int) -> int:
    return ((last // ALIGN + 1) * ALIGN - first // ALIGN * ALIGN) // 32


def _expected(terms, spans, index_bytes, dense_off, dense_bytes, ratio=16.0, budget=2.0):
    """per term the word its probes read (dense offset, probe offset or NONE), the number of probe terms and their bytes"""
    words = [_span_words(*s) if s else 0 for s in spans]
    qual = [t for t in range(len(terms)) if spans[t] and dense_off[t] == NONE and 4 * words[t] <= ratio * int(terms["chunk_len"][t])]
    qual.sort(key=lambda t: -int(terms["documents"][t]))  # stable: ties keep the lower term id first
    off = dense_off.copy()
    base, used, n = dense_bytes // 4, 0, 0
    for t in qual:
        if 4 * (used + words[t]) > budget * index_bytes or base + used + words[t] >= 2**32:
            break
        off[t] = base + used
        used += words[t]
        n += 1
    return off, n, 4 * used


def _index(codec, lists):
    b = tb.IndexBuilder(codec)
    for d in lists:
        b.add_term(d, np.ones(len(d), np.uint32))
    return b.index(), b.terms_array()


def _spans(lists):
    return [(int(d[0]), int(d[-1])) if len(d) else None for d in lists]


NDOCS = 1_000_000


def _lists():
    """densities from every 2nd document to every 20000th: the densest terms get dense bitmaps, the middle probe bitmaps, the sparsest none;
    two terms of equal df; a sparse term inside a narrow span"""
    out = [np.arange(step, NDOCS + 1, step, dtype=np.uint32) for step in (2, 3, 40, 90, 90, 150, 300, 900, 2000, 5000, 20000)]
    out.append(np.arange(700_000, 700_000 + 40 * 2000, 40, dtype=np.uint32))
    return out


def _check(codec, index, terms, lists, **kw):
    dense_off, dense_bytes = tb.debug_dense_terms(codec, index, terms)
    off, n, nbytes = tb.debug_probe_terms(codec, index, terms)
    want = _expected(terms, _spans(lists), index.size, dense_off, dense_bytes, **kw)
    assert np.array_equal(off, want[0]) and (n, nbytes) == want[1:], (kw, off, want)
    return dense_off, dense_bytes, off, n, nbytes


def test_selection(monkeypatch):
    lists = _lists()
    index, terms = _index(G, lists)
    dense_off, dense_bytes, off, n, nbytes = _check(G, index, terms, lists)
    dense = dense_off != NONE
    tier = (off != NONE) & ~dense
    # the tiers do not overlap: a dense term keeps its dense offset, the tier starts where the dense bitmaps end
    assert dense.sum() == 2 and np.array_equal(off[dense], dense_off[dense])
    assert n == tier.sum() > 0 and off[tier].min() == dense_bytes // 4
    # densest first: the offsets grow as df falls, the two terms of equal df in term order; the sparsest term has none
    order = np.flatnonzero(tier)
    assert list(order[np.argsort(off[tier])]) == sorted(order, key=lambda t: (-int(terms["documents"][t]), t))
    assert off[3] < off[4] and off[10] == NONE
    # the ratio decides which terms qualify
    for ratio in (1.0, 4.0, 8.0, 32.0, 1000.0):
        monkeypatch.setenv("TRN_PROBE_RATIO", repr(ratio))
        _check(G, index, terms, lists, ratio=ratio)
    monkeypatch.setenv("TRN_PROBE_RATIO", "1000")
    assert tb.debug_probe_terms(G, index, terms)[1] > n
    monkeypatch.delenv("TRN_PROBE_RATIO")
    # the budget stops the selection part way: it does not skip a term to fit a smaller one behind it
    for budget in (0.01, 0.05, 0.2, 1.0, 5.0):
        monkeypatch.setenv("TRN_PROBE_BUDGET", repr(budget))
        _, _, _, _, b = _check(G, index, terms, lists, budget=budget)
        assert b <= budget * index.size
    first = off[order[np.argmin(off[order])]]
    first_t = int(np.flatnonzero(off == first)[0])
    w0 = 4 * _span_words(*_spans(lists)[first_t])
    monkeypatch.setenv("TRN_PROBE_BUDGET", repr((w0 + ALIGN // 8) / index.size))
    o, k, _ = tb.debug_probe_terms(G, index, terms)
    assert k == 1 and o[first_t] == dense_bytes // 4
    assert tb.debug_probe_terms(G, index, terms)[0][11] == NONE  # the narrow term (one 2^17 tile) would still fit


def test_off_switches_and_lucene(monkeypatch):
    lists = _lists()
    index, terms = _index(G, lists)
    dense_off, _ = tb.debug_dense_terms(G, index, terms)
    for knob, value in (("TRN_PROBE_BITMAPS", "0"), ("TRN_PROBE_BUDGET", "0")):
        with _env({knob: value}):
            off, n, nbytes = tb.debug_probe_terms(G, index, terms)
            assert np.array_equal(off, dense_off) and n == 0 and nbytes == 0, knob
    with _env({"TRN_DENSE_BITMAPS": "0"}):
        off, n, nbytes = tb.debug_probe_terms(G, index, terms)
        assert np.all(off == NONE) and n == 0 and nbytes == 0
    index, terms = _index(L, lists)
    off, n, nbytes = tb.debug_probe_terms(L, index, terms)
    assert np.all(off == NONE) and n == 0 and nbytes == 0


def test_word_cap(monkeypatch):
    """terms whose spans cover the whole docID space (2^27 words each): both tiers together stay below 2^32 words"""
    lists = [np.array([1 + i] + list(range(1000, 1000 + 3 * i, 3)) + [TOP], np.uint32) for i in range(40, 0, -1)]
    index, terms = _index(G, lists)
    monkeypatch.setenv("TRN_PROBE_RATIO", "1e12")
    monkeypatch.setenv("TRN_PROBE_BUDGET", "1e12")
    dense_off, dense_bytes, off, n, nbytes = _check(G, index, terms, lists, ratio=1e12, budget=1e12)
    assert dense_bytes == 0 and n == 31 and nbytes == 31 * 2**29
    assert list(off[:31]) == [k << 27 for k in range(31)] and np.all(off[31:] == NONE)


@pytest.mark.parametrize("first", [TOP - 40 * 2000, 2**32 - ALIGN - 30_000])
def test_span_ending_at_the_top(monkeypatch, first):
    d = np.arange(first, TOP + 1, 40, dtype=np.uint64)
    d = np.append(d[d < TOP], TOP).astype(np.uint32)
    lists = [d, np.array([5, 9], np.uint32)]
    index, terms = _index(G, lists)
    monkeypatch.setenv("TRN_PROBE_BUDGET", "1000")
    dense_off, _, off, n, nbytes = _check(G, index, terms, lists, budget=1000)
    tiles = 1 if first >= 2**32 - ALIGN else 2
    assert dense_off[0] == NONE and off[0] == 0 and off[1] == NONE and n == 1 and nbytes == tiles * ALIGN // 8


def _batches():
    """(label, index, terms, max_docid, plans): the corpora of the candidate-driven edge tests with their queries, and bench.py's and2 and
    tree8 batches on a reduced index"""
    out = []
    corpora = [("lead", cu.lead_corpus(), cu.lead_queries() + cu.mixed_lead_queries()), ("probe", cu.probe_corpus(), cu.PROBE_QUERIES),
               ("truth", cu.truth_corpus(), cu.all_truth_queries()), ("group", cu.group_corpus(), [(q, 0, 0) for q in cu.GROUP_ROUTES]),
               ("top", cu.top_corpus(), cu.TOP_QUERIES)]
    for label, lists, qs in corpora:
        index, terms, names = cu.build(lists)
        mx = int(max(int(v[-1]) for v in lists.values()))
        out.append((label, index, terms, mx, cu.parse(qs, tb.TermDictionary(names))))
    ndocs, nterms = 2_000_000, 512
    s = tb.SynthIndex(G, ndocs, nterms, threads=2)
    tdict = tb.TermDictionary(s.names)
    for w in ("and2", "tree8"):
        texts, _ = bench.gen_queries(w, 300, nterms)
        out.append((w, np.array(s.index), np.array(s.terms), ndocs, [tb.parse_query(q, tdict) for q in texts]))
    return out


def _planned(index, terms, mx, plans, mode):
    routes, slots = tb.debug_plan(G, index, terms, plans, mode, max_docid=mx)
    runs = [fn(G, index, terms, plans, mode, max_docid=mx) for fn in (tb.debug_dense_runs, tb.debug_mixed_runs, tb.debug_cand_runs)]
    return list(routes), tuple(slots), [(q.tolist(), t.tolist()) for q, t in runs], tb.debug_dense_terms(G, index, terms)


@pytest.mark.parametrize("cost", [None, "1"])
def test_plans_unchanged(cost):
    """routes, slot counts, the dense, mixed and candidate run tickets and the dense selection: the same with the tier off, on by default
    and at the largest ratio and budget"""
    base = {} if cost is None else {"TRN_CAND_COST": cost}
    for label, index, terms, mx, plans in _batches():
        with _env({**base, "TRN_PROBE_BITMAPS": "0"}):
            off = {m: _planned(index, terms, mx, plans, m) for m in (tb.MODE_DOCS_ONLY, tb.MODE_DOCS_COMPACT)}
            assert tb.debug_probe_terms(G, index, terms)[1] == 0
        for env in ({}, {"TRN_PROBE_RATIO": "1e9", "TRN_PROBE_BUDGET": "1e9"}):
            with _env({**base, **env}):
                assert tb.debug_probe_terms(G, index, terms)[1] > 0 or not env, label
                for m, want in off.items():
                    got = _planned(index, terms, mx, plans, m)
                    assert got[:3] == want[:3], (label, env, m)
                    assert np.array_equal(got[3][0], want[3][0]) and got[3][1] == want[3][1], (label, env, m)
