"""The default exec mode (TRN_MODE_MATCHED_TERMS) on the CPU: the host encoders' payload bytes against the reference Encoder's, the
kernels' hit walker (trn_debug_hits) against the reference's materialize_hits, the collect rules (matchutil.restated_terms) against the
reference's exec_query with no ExecFlags, and the planner's view of the mode (trn_debug_plan)."""
import numpy as np
import pytest

import trinity_b200 as tb
from matchutil import doc_corpus, host_build, lists_from, payload_hits, ref_build, restated_terms
from test_frontend_cpu import EXTRA, OPTIONAL_QUERIES, SOME_QUERIES
from test_gpu_parity import TEMPLATES
from test_phrase_cpu import QUERIES as PHRASE_QUERIES

CODECS = [tb.CODEC_GOOGLE, tb.CODEC_LUCENE]
IDS = ["google", "lucene"]


def edge_lists(rng):
    """term-major lists that reach the LUCENE layout's edges: full 128-hit blocks, documents whose hits cross blocks and reach the tail,
    freq-0 documents, every payload size 0..8 (growing and shrinking inside a document) and 1000-hit documents"""
    per = []
    for t, (ndocs, fmax) in enumerate([(300, 3), (40, 300), (200, 20), (5, 1000), (130, 1)]):
        d = {}
        docs = np.sort(rng.choice(np.arange(1, 5000), size=ndocs, replace=False))
        for x in docs:
            f = int(rng.integers(1, fmax + 1))
            d[int(x)] = sorted(int(p) for p in rng.integers(1, 8192, size=f))
        per.append(d)
    lists, _ = lists_from(rng, per)
    # freq-0 documents (a document with no hits) in a term of each shape
    out = []
    for docs, freqs, pos, sz, pv in lists:
        z = rng.random(len(docs)) < 0.1
        keep = np.repeat(~z, freqs)
        out.append((docs, np.where(z, 0, freqs).astype(np.uint32), pos[keep], sz[keep], pv[keep]))
    return out


@pytest.fixture(scope="module")
def edges():
    rng = np.random.default_rng(5)
    lists = edge_lists(rng)
    names = [f"e{i + 1}" for i in range(len(lists))]
    return lists, names


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_host_encoder_payload_bytes_equal_the_reference_encoder(edges, codec):
    lists, names = edges
    index, hits, terms = host_build(codec, lists)
    r = ref_build(codec, lists, names, 5000)
    assert np.array_equal(terms, r.terms())
    for mine, theirs in ((index, r.index()), (hits, r.hits())):
        assert mine.size == theirs.size
        diff = np.flatnonzero(mine != theirs)
        # LUCENE: only the padding bytes the reference's FastPFor leaves uninitialised (fastpfor.h:196-198) may differ; ours are 0
        assert diff.size == 0 if codec == tb.CODEC_GOOGLE else (np.all(mine[diff] == 0) and diff.size < max(mine.size // 50, 8)), diff[:10]
    # every payload size occurs, and so do size changes inside a document
    sz = np.concatenate([l[3] for l in lists])
    assert set(np.unique(sz).tolist()) == set(range(9))


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_debug_hits_equal_the_reference_hits(edges, codec):
    lists, names = edges
    index, hits, terms = host_build(codec, lists)
    r = ref_build(codec, lists, names, 5000)
    for t, name in enumerate(names):
        want = {d: ts[0] for d, ts in r.exec(name)}
        docs = lists[t][0]
        probe = np.concatenate([docs, docs[:20] + 1]).astype(np.uint32)  # + documents the term may not hold
        got = tb.debug_hits(codec, index, hits, terms[t], probe)
        for d, g in zip(probe.tolist(), got):
            if d not in want:
                assert g is None or d in set(docs.tolist()), (name, d)
                continue
            _, wf, wp, wl, wv = want[d]
            assert g is not None and g[0] == wf, (name, d)
            assert np.array_equal(g[1].astype(np.uint16), wp), (name, d)
            assert np.array_equal(g[2], wl), (name, d)
            assert np.array_equal(g[3], wv), (name, d)
    if codec == tb.CODEC_LUCENE:  # a freq-0 document is held, with no hits
        zero = [(t, int(d)) for t, l in enumerate(lists) for d, f in zip(l[0], l[1]) if f == 0]
        assert zero
        t, d = zero[0]
        assert tb.debug_hits(codec, index, hits, terms[t], [d])[0][0] == 0


@pytest.fixture(scope="module")
def text(request):
    rng = np.random.default_rng(11)
    lists, positions = doc_corpus(rng, 3000, 10)
    names = [f"t{i + 1}" for i in range(10)]
    return lists, positions, names


ROOT_NOT = ["(t1 OR t2) NOT t3", "(t4 OR t5) NOT t1", "(t2 OR t3 OR t6) NOT t4 NOT t5"]
MORE = ["t1 AND t1", "t1 OR t1 OR t2", "t4 NOT (t1 AND t2)", "t5 AND nosuchterm", "t6 OR nosuchterm", "t7 NOT nosuchterm"]
# (a MatchSome group whose min exceeds its size, ("[t1, t2]", 3), crashes the reference in this mode: left out of the comparison)
SOME_DEFAULT = [(q, m) for q, m in SOME_QUERIES if (q, m) != ("[t1, t2]", 3)]
CASES = ([(q, 0, 0) for q in TEMPLATES + EXTRA + ROOT_NOT + MORE] + [(q, 8, 0) for q in OPTIONAL_QUERIES] + [(q, 16, m) for q, m in SOME_DEFAULT]
         + [(q.replace("w", "t"), 0, 0) for q in PHRASE_QUERIES])


@pytest.mark.parametrize("q,flags,m", CASES)
def test_collect_rules_restated_equal_the_reference(text, q, flags, m):
    lists, positions, names = text
    r = ref_build(tb.CODEC_GOOGLE, lists, names, 3000)
    want = {d: frozenset(t for t, *_ in ts) for d, ts in r.exec(q, flags, m)}
    nodes = tb.parse_query(q, tb.TermDictionary(names), min_match=m or None)
    got = restated_terms(nodes, lists, positions, 3000)
    assert got == want, q


def test_root_filter_over_a_disjunction_excludes_in_the_default_mode(text):
    """(a OR b) NOT c with df(c) <= df(a) + df(b): DocumentsOnly keeps c's documents (the reference quirk), the default mode excludes them"""
    lists, positions, names = text
    r = ref_build(tb.CODEC_GOOGLE, lists, names, 3000)
    q = "(t1 OR t2) NOT t3"
    assert len(lists[2][0]) <= len(lists[0][0]) + len(lists[1][0])
    got = {d for d, _ in r.exec(q)}
    c = set(lists[2][0].tolist())
    assert got and not (got & c)
    ab = set(lists[0][0].tolist()) | set(lists[1][0].tolist())
    assert got == ab - c


def _plan_routes(codec, index, terms, qs, mode):
    return tb.debug_plan(codec, index, terms, qs, mode)[0]


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_debug_plan_routes_and_limits(text, codec):
    lists, positions, names = text
    index, hits, terms = host_build(codec, lists)
    tdict = tb.TermDictionary(names)
    plain = [q for q in TEMPLATES + EXTRA if q != "t1 | t9 -t3"]  # (that one is a root filter over a disjunction: below)
    qs = [tb.parse_query(q, tdict) for q in plain]
    if codec == tb.CODEC_LUCENE:  # no hits.data on the planner's side: refused like a phrase plan
        with pytest.raises(tb.TrinityError, match="hits"):
            tb.debug_plan(codec, index, terms, qs, tb.MODE_MATCHED_TERMS)
        return
    got = _plan_routes(codec, index, terms, qs, tb.MODE_MATCHED_TERMS)
    want = _plan_routes(codec, index, terms, qs, tb.MODE_DOCS_ONLY)
    assert np.array_equal(got, want)
    # a root filter over a disjunction: DocumentsOnly runs the bare disjunction (the reference quirk), this mode the whole filter
    q = [tb.parse_query("(t1 OR t9) NOT t3", tdict)]
    assert _plan_routes(codec, index, terms, q, tb.MODE_DOCS_ONLY)[0] == tb.ROUTE_FLAT_OR
    assert _plan_routes(codec, index, terms, q, tb.MODE_MATCHED_TERMS)[0] != tb.ROUTE_FLAT_OR
    # 32 distinct terms are taken, 33 are refused
    many = [(np.arange(1, 50, dtype=np.uint32) * (i + 1), np.ones(49, np.uint32)) for i in range(40)]
    b = tb.IndexBuilder(codec)
    for d, f in many:
        b.add_term(d, f)
    idx2, t2 = b.index(), b.terms_array()
    td = tb.TermDictionary([f"m{i}" for i in range(40)])
    q32 = tb.parse_query(" OR ".join(f"m{i}" for i in range(32)), td)
    q33 = tb.parse_query(" OR ".join(f"m{i}" for i in range(33)), td)
    tb.debug_plan(codec, idx2, t2, [q32], tb.MODE_MATCHED_TERMS)
    with pytest.raises(tb.TrinityError, match="32 distinct terms"):
        tb.debug_plan(codec, idx2, t2, [q33], tb.MODE_MATCHED_TERMS)
