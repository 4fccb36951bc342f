"""Flat-tree plans (planner.cpp flat_tree_transform, exec_docs_flat.cuh tree_exec_google) on the device vs the reference's exec_query: a
skewed vocabulary (df from 20 to half of the documents), so that the leaves of one tree have very unequal block counts; every tree shape
of the benchmark plus nested ones, random term choices; documents bit-exact.  With TRN_CAND_COST=0 (every tree but the plain
conjunctions on the flat-tree path), in the default configuration, and for a source that does not start at docID 1 (a shard)."""
import os

import numpy as np
import pytest

import trinity_b200 as tb
from refharness import RefIndex
from test_plan_compiler_cpu import TREE8
from util import assert_same_docs

pytestmark = pytest.mark.gpu
NDOCS = 600_000
DFS = [300_000, 200_000, 120_000, 40_000, 12_000, 4_000, 1_400, 400, 100, 20, 180_000, 6_000]
FLAT_TREES = 200  # of the 225 queries with TRN_CAND_COST=0: all but the 25 two-term conjunctions, which take the flat AND (tb.debug_plan)


def _corpus(ref, lo=1):
    rng = np.random.default_rng(78)
    lists = []
    for df in DFS:
        d = np.sort(rng.choice(NDOCS - lo + 1, size=min(df, NDOCS - lo + 1), replace=False).astype(np.uint32) + lo)
        lists.append((d, rng.integers(1, 4, size=len(d)).astype(np.uint32)))
    names = [f"t{i + 1}" for i in range(len(lists))]
    r = RefIndex(ref, tb.CODEC_GOOGLE)
    b = tb.IndexBuilder(tb.CODEC_GOOGLE)
    for n, (d, f) in zip(names, lists):
        r.add_term(n, d, f)
        b.add_term(d, f)
    r.finish(NDOCS)
    return r, b, names


@pytest.mark.parametrize("lo", [1, 250_001], ids=["whole", "shard"])
def test_flat_tree_matches_reference(ref, lo):
    r, b, names = _corpus(ref, lo)
    tdict = tb.TermDictionary(names)
    rng = np.random.default_rng(9)
    qs = []
    for _ in range(25):
        for tpl in TREE8:
            pick = rng.choice(len(names), size=8, replace=False)
            qs.append(tpl.format(*[names[i] for i in pick]))
    plans = [tb.parse_query(q, tdict) for q in qs]
    want = [r.exec(q, False, NDOCS + 1)[0] for q in qs]
    os.environ["TRN_CAND_COST"] = "0"  # the candidate-driven path would take most of these: keep them on the flat-tree path
    try:
        g = tb.GpuIndexSource(0)
        g.upload(tb.CODEC_GOOGLE, b.index(), b.terms_array(), NDOCS)
        res = g.exec_batch(plans, tb.MODE_DOCS_ONLY)
        assert int(np.count_nonzero(g.last_routes() == tb.ROUTE_FLAT_TREE)) == FLAT_TREES
        for i, q in enumerate(qs):
            assert_same_docs(res.query(i)[0], want[i], f"[{q}] TRN_CAND_COST=0 lo={lo}")
        g.close()
    finally:
        del os.environ["TRN_CAND_COST"]
    # default configuration (candidate-driven where it pays)
    g = tb.GpuIndexSource(0)
    g.upload(tb.CODEC_GOOGLE, b.index(), b.terms_array(), NDOCS)
    res = g.exec_batch(plans, tb.MODE_DOCS_ONLY)
    for i, q in enumerate(qs):
        assert_same_docs(res.query(i)[0], want[i], f"[{q}] default lo={lo}")
    g.close()
