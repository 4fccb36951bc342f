"""TRN_MODE_DOCS_COMPACT on the device: the same DocumentsOnly plans, results leaving the GPU as per-tile bitmaps / 16-bit offsets /
docIDs (whichever is smallest), replayed on the host by trn_result_decode — must equal the plain DocumentsOnly stream and the reference's
exec_query, on every path of k_exec_docs (GOOGLE: step programs, flat AND/OR and flat-tree plans in the first test, candidate-driven plans
in the second; LUCENE: step programs — asserted through GpuIndexSource.last_routes), through the pipelined call (large batch) and the
single-call form (small batch), with masked documents, and for a docID-range shard."""
import numpy as np
import pytest

import trinity_b200 as tb
from refharness import RefIndex
from test_frontend_cpu import EXTRA, OPTIONAL_QUERIES
from test_gpu_parity import TEMPLATES
from test_plan_compiler_cpu import TREE8
from util import assert_same_docs, closed_form_lists

pytestmark = pytest.mark.gpu
NDOCS = 400_000


def _index(codec, lists):
    b = tb.IndexBuilder(codec)
    for d, f in lists:
        b.add_term(d, f)
    g = tb.GpuIndexSource(0)
    g.upload(codec, b.index(), b.terms_array(), NDOCS)
    return g


@pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def test_compact_equals_plain_and_reference(ref, codec):
    lists = closed_form_lists(NDOCS)
    names = [f"t{i + 1}" for i in range(len(lists))]
    tdict = tb.TermDictionary(names)
    r = RefIndex(ref, codec)
    for n, (d, f) in zip(names, lists):
        r.add_term(n, d, f)
    r.finish(NDOCS)
    g = _index(codec, lists)
    qs = [q for q in TEMPLATES + EXTRA if "nosuchterm" not in q]
    nplain = len(qs)
    qs += OPTIONAL_QUERIES  # (the reference parses '<t>' as optional only with parser flag 8)
    rng = np.random.default_rng(4)
    for tpl in TREE8:
        for _ in range(3):
            qs.append(tpl.format(*[names[i] for i in rng.choice(len(names), size=8, replace=False)]))
    plans = [tb.parse_query(q, tdict) for q in qs]
    flags = [8 if nplain <= i < nplain + len(OPTIONAL_QUERIES) else 0 for i in range(len(qs))]
    want = [r.exec(q, False, NDOCS + 1, parser_flags=f)[0] for q, f in zip(qs, flags)]
    encodings = set()
    for batch in (plans, plans[:5]):  # pipelined call (>= 32 queries) and the single-call form
        plain = g.exec_batch(batch, tb.MODE_DOCS_ONLY)
        routes = set(g.last_routes().tolist())
        comp = g.exec_batch(batch, tb.MODE_DOCS_COMPACT, copy=False)
        assert set(g.last_routes().tolist()) == routes
        if batch is plans:  # the paths this test claims to cover were taken
            want_routes = {tb.ROUTE_STEPS, tb.ROUTE_FLAT_AND, tb.ROUTE_FLAT_OR, tb.ROUTE_FLAT_TREE} if codec == tb.CODEC_GOOGLE else {tb.ROUTE_STEPS}
            assert routes >= want_routes if codec == tb.CODEC_GOOGLE else routes == want_routes, routes
        assert np.array_equal(comp.match_counts, plain.match_counts)
        assert comp.result_bytes() <= plain.result_bytes() + 4 * comp.nitems
        desc = np.ctypeslib.as_array(comp.raw.item_desc, shape=(max(comp.nitems, 1),))[: comp.nitems]
        encodings |= set(int(x) >> 30 for x in desc if int(x) & 0x3FFFFFFF)
        for i in range(len(batch)):
            got = comp.decode_query(i)
            assert_same_docs(got, plain.query(i)[0], f"[{qs[i]}] compact vs plain")
            assert_same_docs(got, want[i], f"[{qs[i]}] compact vs reference")
        assert np.array_equal(comp.checksums(), plain.checksums())
    assert encodings >= {1, 2, 3}, encodings  # 16-bit offsets, bitmaps and bucketed 8-bit offsets all occurred
    # decoded copy (copy=True) behaves like a plain result
    dec = g.exec_batch(plans, tb.MODE_DOCS_COMPACT)
    for i in (0, 7, len(plans) - 1):
        assert_same_docs(dec.query(i)[0], want[i], f"[{qs[i]}] decoded copy")
    # masked documents never reach the sink in either form
    masked = np.unique(np.random.default_rng(5).integers(1, NDOCS + 1, 9000)).astype(np.uint32)
    g.set_masked_documents(masked)
    plain = g.exec_batch(plans, tb.MODE_DOCS_ONLY)
    comp = g.exec_batch(plans, tb.MODE_DOCS_COMPACT, copy=False)
    for i in range(0, len(plans), 3):
        assert_same_docs(comp.decode_query(i), plain.query(i)[0], f"[{qs[i]}] masked")
        assert not np.isin(comp.decode_query(i), masked).any()
    g.close()


def test_compact_sparse_results_and_a_shard(ref):
    """rare terms (candidate-driven path: docID lists) and a source whose docIDs start far from 1"""
    rng = np.random.default_rng(12)
    lo = 2_600_000
    ndocs = 3_000_000
    dfs = [200_000, 150_000, 30_000, 3_000, 300, 40, 90_000, 1_000]
    lists = []
    for df in dfs:
        d = np.sort(rng.choice(ndocs - lo, size=df, replace=False).astype(np.uint32) + lo + 1)
        lists.append((d, np.ones(df, np.uint32)))
    names = [f"t{i + 1}" for i in range(len(lists))]
    tdict = tb.TermDictionary(names)
    r = RefIndex(ref, tb.CODEC_GOOGLE)
    b = tb.IndexBuilder(tb.CODEC_GOOGLE)
    for n, (d, f) in zip(names, lists):
        r.add_term(n, d, f)
        b.add_term(d, f)
    r.finish(ndocs)
    g = tb.GpuIndexSource(0)
    g.upload(tb.CODEC_GOOGLE, b.index(), b.terms_array(), ndocs)
    qs = ["t1 AND t2", "t1 AND t5", "t4 AND t6", "t1 OR t2", "t3 AND (t1 OR t2)", "(t1 AND t2) OR (t3 AND t7)", "t1 AND t2 AND t7", "t1 NOT t2", "t6", "t1"] * 4
    plans = [tb.parse_query(q, tdict) for q in qs]
    comp = g.exec_batch(plans, tb.MODE_DOCS_COMPACT, copy=False)
    assert tb.ROUTE_CANDIDATE in g.last_routes().tolist()
    for i, q in enumerate(qs[:10]):
        assert_same_docs(comp.decode_query(i), r.exec(q, False, ndocs + 1)[0], f"[{q}] shard")
    g.close()
