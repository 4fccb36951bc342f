"""Phrases of up to 16 terms on the device, on every path that checks positions.  The corpus and the queries are
test_phrase_edges_cpu's (which pins their planted answers, the OP_ARG packing and the position cursors on the CPU).

§1 result modes (test_result_modes), GOOGLE and LUCENE (with its hits.data), each with and without payloads:
  k_exec_docs<PH> (exec_docs.cuh) in MODE_DOCS_ONLY and MODE_DOCS_COMPACT, docIDs bit-exact; k_exec_tiles<PH> (kernels.cu) in
  MODE_SCORED_ALL within 1e-5 and MODE_SCORED_TOPK at k = 1, 25, 512.  Both reach phrase_match_count (phrase.cuh), whose phrase_arg reads
  term j from the (j >> 2)-th OP_ARG step, and the cursors of hitcursor.h (GOOGLE inline payload bytes skipped by `p += psize`, LUCENE tail
  size bytes by `++p`).  The route of every query is asserted.
§2 the default exec mode's collect pass (collect.cuh) on the payload twin: exec_matches against the planted matches (the terms by
  collect_doc_matching_terms' rules, matchutil.restated_terms), hits and payloads bit for bit, with two 16-term phrases of 32 distinct terms in one query; a 33rd distinct term is refused (test_payload_twin_matches).
§3 configurations: TRN_DOCS_SHIFT 13 / 14 / 17, masked documents, a pipelined batch of >= 64 queries under TRN_PIPELINE_CHUNKS=8, the
  corpus translated to end at docID 2^32 - 2, and the phrases beside all-bitmap, flat AND, flat OR and flat-tree plans in one batch (whose
  results must equal those of their own batch: a phrase takes them off the run-major tickets).
§4 the percolator's perc_phrase (percolate.cuh) with the anchor at index 0, in the middle and at k - 1, against RefPercolator.
§5 phrases of 1 and 17 terms built by hand are refused by exec_batch, exec_matches and percolator_register, and the context still answers.

The oracle is test_phrase_edges_cpu's restatement (pyeval.evaluate, whose structural rules and phrase scoring are pinned against the
reference's exec_query in test_phrase_cpu), which equals the planted answers; the reference's own exec_query was not stable on this corpus.
"""
import contextlib
import os

import numpy as np
import pytest

import trinity_b200 as tb
from matchutil import assert_same_matches, gpu_as_list, host_build, restated_terms
from percutil import RefPercolator
from test_phrase_edges_cpu import (_POS, NAMES, NDOCS, OTHERS, PERC_PHRASES, TEXTS, V, WANT, build, hand_phrase, lists, payload_lists,
                                   perc_costs, perc_docs, restated, tdict, text)
from util import assert_close_scores, assert_same_docs, assert_topk_equal

pytestmark = pytest.mark.gpu

G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE
TOP = 2**32 - 2
DELTA = TOP - NDOCS
KS = [1, 25, 512]


@contextlib.contextmanager
def _env(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k)
            else:
                os.environ[k] = v


class Oracle:
    """the restated answers (test_phrase_edges_cpu.restated: pyeval.evaluate, equal to the planted ones), cached per query"""

    def __init__(self):
        self.cache = {}

    def __call__(self, q, scored=False, masked=None):
        if q not in self.cache:
            m, sc = restated(q)
            d = np.flatnonzero(m).astype(np.uint32)
            self.cache[q] = (d, sc[d])
        d, sc = self.cache[q]
        if masked is not None:  # a masked document is dropped before it is scored; the others keep their scores
            keep = ~np.isin(d, masked)
            d, sc = d[keep], sc[keep]
        return d, (sc if scored else None)


@pytest.fixture(scope="module")
def oracle():
    o = Oracle()
    for q, w in zip(TEXTS, WANT):  # (pinned on the CPU too)
        assert np.array_equal(o(q)[0], w), q
    return o


_BUILT = {}


def _built(codec, payloads):
    if (codec, payloads) not in _BUILT:
        _BUILT[(codec, payloads)] = host_build(codec, payload_lists()) if payloads else build(codec)
    return _BUILT[(codec, payloads)]


def _source(codec, payloads=False, env=None, ls=None, max_docid=NDOCS):
    index, hits, terms = build(codec, ls) if ls is not None else _built(codec, payloads)
    with _env(env or {}):
        g = tb.GpuIndexSource(0)
    g.upload(codec, index, terms, max_docid)
    if codec == L:
        g.upload_hits(index, hits)
    return g


def _plans(scored, g=None, texts=TEXTS):
    out = [tb.parse_query(q, tdict()) for q in texts]
    if scored:
        for p in out:
            g.set_bm25_weights(p, NDOCS)
    return out


def _docs_modes(g, oracle, label, texts=TEXTS, masked=None, shift=0):
    plans = _plans(False, texts=texts)
    res = g.exec_batch(plans, tb.MODE_DOCS_ONLY)
    assert g.last_routes().tolist() == [tb.ROUTE_STEPS] * len(plans), label
    comp = g.exec_batch(plans, tb.MODE_DOCS_COMPACT, copy=False)
    for n, q in enumerate(texts):
        want = (oracle(q, False, masked)[0].astype(np.uint64) + shift).astype(np.uint32)
        assert_same_docs(res.query(n)[0], want, f"{label} [{q}] docs-only")
        assert_same_docs(comp.decode_query(n), want, f"{label} [{q}] compact")


def _scored_modes(g, oracle, label, texts=TEXTS, masked=None, shift=0, ks=KS):
    plans = _plans(True, g, texts)
    res = g.exec_batch(plans, tb.MODE_SCORED_ALL)
    assert g.last_routes().tolist() == [tb.ROUTE_EXEC_TILES] * len(plans), label
    tops = {k: g.exec_batch(plans, tb.MODE_SCORED_TOPK, k=k) for k in ks}
    for n, q in enumerate(texts):
        wd, ws = oracle(q, True, masked)
        wd = (wd.astype(np.uint64) + shift).astype(np.uint32)
        gd, gs = res.query(n)
        assert_same_docs(gd, wd, f"{label} [{q}] scored")
        assert_close_scores(gs, ws, f"{label} [{q}]")
        for k, t in tops.items():
            td, ts = t.query(n)
            assert_topk_equal(td, ts, wd, ws, k, f"{label} [{q}] top-{k}")


# ------------------------------------------------------------------------------------------------ §1 result modes
@pytest.mark.parametrize("payloads", [False, True], ids=["plain", "payloads"])
@pytest.mark.parametrize("codec", [G, L], ids=["google", "lucene"])
def test_result_modes(oracle, codec, payloads):
    g = _source(codec, payloads)
    label = f"codec {codec} payloads {payloads}"
    _docs_modes(g, oracle, label)
    _scored_modes(g, oracle, label)
    g.close()


# ------------------------------------------------------------------------------------------------ §2 the collect pass
_PAY = {}


def _google_payloads(sz, pv):
    """GOOGLE's materialize_hits: the payload starts at 0 in each document, a size of 0 zeroes it, a non-zero size overwrites its low
    bytes — a hit keeps the high bytes of an earlier, longer payload of its document (hitcursor.h HitWalker)"""
    out, cur = np.zeros(len(pv), np.uint64), 0
    for n, (s, v) in enumerate(zip(sz.tolist(), pv.tolist())):
        cur = 0 if s == 0 else (cur & ~((1 << (8 * s)) - 1) & (2**64 - 1)) | v
        out[n] = cur
    return out


def _want_matches(q, codec):
    """the default exec mode's answer by construction: per match (matchutil.restated_terms: collect_doc_matching_terms' rules) every
    collected term with its freq, positions, payload lengths and payloads"""
    if "pay" not in _PAY:
        _PAY["pay"] = payload_lists()
    pay = _PAY["pay"]
    out = []
    for d, ts in sorted(restated_terms(tb.parse_query(q, tdict()), pay, _POS, NDOCS).items()):
        row = []
        for t in sorted(ts):
            ds, fs, ps, sz, pv = pay[t]
            if t not in _PAY:
                _PAY[t] = np.concatenate([[0], np.cumsum(fs.astype(np.int64))])
            n = int(np.searchsorted(ds, d))
            at, f = int(_PAY[t][n]), int(fs[n])
            vals = _google_payloads(sz[at:at + f], pv[at:at + f]) if codec == G else pv[at:at + f]
            row.append((t, f, ps[at:at + f].astype(np.uint16), sz[at:at + f], vals))
        out.append((d, row))
    return out


@pytest.mark.parametrize("codec", [G, L], ids=["google", "lucene"])
def test_payload_twin_matches(oracle, codec):
    g = _source(codec, True)
    res = g.exec_matches(_plans(False))
    for n, q in enumerate(TEXTS):
        want = _want_matches(q, codec)
        assert [d for d, _ in want] == oracle(q)[0].tolist(), q
        assert_same_matches(gpu_as_list(res, n), want, f"codec {codec} [{q}]")
    assert int(res.query(len(TEXTS) - 1).size) > 0  # the query of 32 distinct terms matches
    with pytest.raises(tb.TrinityError, match="32 distinct terms"):
        g.exec_matches([tb.parse_query(TEXTS[-1] + " AND f1", tdict())])
    g.close()


# ------------------------------------------------------------------------------------------------ §3 configurations
@pytest.mark.parametrize("docs_shift", [13, 14, 17])
@pytest.mark.parametrize("codec", [G, L], ids=["google", "lucene"])
def test_docs_shift(oracle, codec, docs_shift):
    g = _source(codec, env={"TRN_DOCS_SHIFT": str(docs_shift)})
    texts = TEXTS
    if docs_shift == 17:  # a slot of a 2^17-docID tile takes 16 KB: the trees' slots do not fit on an SM, and the engine says so
        texts = [q for q in TEXTS if q.count('"') == 2 and " AND " not in q and " NOT " not in q]
        with pytest.raises(tb.TrinityError, match="does not fit on an SM"):
            g.exec_batch(_plans(False, texts=[TEXTS[-2]]), tb.MODE_DOCS_ONLY)
    _docs_modes(g, oracle, f"codec {codec} shift {docs_shift}", texts=texts)
    g.close()


@pytest.mark.parametrize("codec", [G, L], ids=["google", "lucene"])
def test_masked_documents(oracle, codec):
    masked = np.array(sorted({int(w[x]) for w in WANT for x in range(0, len(w), 3)}), np.uint32)  # a third of every answer
    g = _source(codec)
    g.set_masked_documents(masked)
    _docs_modes(g, oracle, f"codec {codec} masked", masked=masked)
    _scored_modes(g, oracle, f"codec {codec} masked", masked=masked, ks=[25])
    g.close()


@pytest.mark.parametrize("codec", [G, L], ids=["google", "lucene"])
def test_pipelined(oracle, codec):
    env = {"TRN_PIPELINE_CHUNKS": "8", "TRN_CHUNK_POSTINGS": "1", "TRN_CHUNK_RULE": "postings"}
    texts = TEXTS * 3
    assert len(texts) >= 64
    with _env(env):
        g = _source(codec, env=env)
        _docs_modes(g, oracle, f"codec {codec} pipelined", texts=texts)
        g.close()


@pytest.mark.parametrize("codec", [G, L], ids=["google", "lucene"])
def test_top_of_the_docid_space(oracle, codec):
    g = _source(codec, ls=lists(DELTA), max_docid=TOP)
    _docs_modes(g, oracle, f"codec {codec} top", shift=DELTA)
    _scored_modes(g, oracle, f"codec {codec} top", shift=DELTA, ks=[25])
    g.close()


def test_mixed_batch(oracle):
    g = _source(G)
    others = _plans(False, texts=OTHERS)
    alone = g.exec_batch(others, tb.MODE_DOCS_ONLY)
    alone_docs = [alone.query(n)[0].copy() for n in range(len(OTHERS))]
    alone_routes = g.last_routes().tolist()
    mixed = _plans(False)[:]
    order = [("p", n) for n in range(len(TEXTS))]
    for n in range(len(OTHERS)):  # interleaved
        mixed.insert(2 * n + 1, others[n])
        order.insert(2 * n + 1, ("o", n))
    res = g.exec_batch(mixed, tb.MODE_DOCS_ONLY)
    routes = g.last_routes().tolist()
    for at, (kind, n) in enumerate(order):
        got = res.query(at)[0]
        if kind == "o":
            assert routes[at] == alone_routes[n], OTHERS[n]
            assert_same_docs(got, alone_docs[n], f"[{OTHERS[n]}] beside the phrases vs in its own batch")
            assert_same_docs(got, oracle(OTHERS[n])[0], f"[{OTHERS[n]}] beside the phrases")
        else:
            assert routes[at] == tb.ROUTE_STEPS
            assert_same_docs(got, oracle(TEXTS[n])[0], f"[{TEXTS[n]}] beside flat plans")
    g.close()


# ------------------------------------------------------------------------------------------------ §4 the percolator
def test_percolator_phrases():
    plans = [tb.parse_query(text(ph), tdict()) for ph in PERC_PHRASES]
    docs = perc_docs()
    want = RefPercolator([(text(ph), 0, 0) for ph in PERC_PHRASES], vocab=NAMES).run(docs)
    for cost in perc_costs():
        p = tb.Percolator(plans, nterms=V, term_cost=cost)
        r = p.percolate(docs)
        for n, w in enumerate(want):
            assert r.document(n).tolist() == w.tolist(), (n, docs[n].tolist())


# ------------------------------------------------------------------------------------------------ §5 refusals
def test_phrases_of_1_and_17_terms_are_refused(oracle):
    g = _source(G)
    good = _plans(False)
    before = g.exec_batch(good, tb.MODE_DOCS_ONLY)
    before = [before.query(n)[0].copy() for n in range(len(good))]
    for n in (1, 17):
        bad = hand_phrase(n)
        with pytest.raises(tb.TrinityError, match="2..16 terms"):
            g.exec_batch([good[0], bad], tb.MODE_DOCS_ONLY)
        with pytest.raises(tb.TrinityError, match="2..16 terms"):
            g.exec_matches([bad])
        with pytest.raises(tb.TrinityError, match="2..16 terms"):
            g.percolator_register([bad], V)
        after = g.exec_batch(good, tb.MODE_DOCS_ONLY)
        for q in range(len(good)):
            assert_same_docs(after.query(q)[0], before[q], f"[{TEXTS[q]}] after a refusal")
    for q in range(len(good)):
        assert_same_docs(before[q], oracle(TEXTS[q])[0], TEXTS[q])
    g.close()
