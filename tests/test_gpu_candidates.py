"""Candidate-driven conjunctions (exec_docs_cand.cuh == the leap-frog of DocsSetIterators::Conjuction, docset_iterators.cpp:282-348)
against the reference exec_query — forced on for every all-term AND (TRN_CAND_COST=1), and compared with the bitmap path (=0)."""
import os

import numpy as np
import pytest

import trinity_b200 as tb
from test_frontend_cpu import EXTRA, OPTIONAL_QUERIES, SOME_QUERIES, TEMPLATES
from util import Pair, assert_same_docs, closed_form_lists

pytestmark = pytest.mark.gpu
NDOCS = 2_000_000


def make_lists(seed=11):
    rng = np.random.default_rng(seed)
    lists = []
    # densities from every second document to one in 50 000 (gaps >= 16384: 3-byte varbyte codes leave the staged block head)
    for p in (0.5, 0.2, 0.05, 0.01, 0.002, 0.0004, 0.00002):
        n = max(3, int(NDOCS * p))
        d = np.sort(rng.choice(np.arange(1, NDOCS + 1), size=n, replace=False)).astype(np.uint32)
        lists.append((d, rng.integers(1, 5, size=n).astype(np.uint32)))
    # blocks whose doc-delta section starts with 3-byte codes and then runs past the 80 staged bytes (10 x 3 + 21 x 2 = 72 bytes + up to
    # 15 bytes of alignment): the lead decoder has to leave its shared-memory slot in the middle of the 2-byte codes
    gaps = np.tile(np.array([16400] * 10 + [130] * 22, np.uint64), 11)
    d = np.cumsum(gaps).astype(np.uint32)
    assert d[-1] <= NDOCS
    lists.append((d, np.ones(len(d), np.uint32)))
    # a term of exactly 32*k documents and one with a 1-document last block
    lists.append((np.arange(7, 7 + 64 * 1000, 1000, dtype=np.uint32), np.ones(64, np.uint32)))
    lists.append((np.arange(3, 3 + 33 * 5, 5, dtype=np.uint32), np.ones(33, np.uint32)))
    return lists


QUERIES = ["t1 AND t2", "t1 AND t5", "t2 AND t6", "t1 AND t7", "t3 AND t4", "t4 AND t5", "t5 AND t6", "t6 AND t7", "t1 AND t2 AND t3",
           "t1 AND t4 AND t6", "t2 AND t3 AND t4 AND t5", "t1 AND t8", "t2 AND t9", "t8 AND t9", "t1 AND nosuchterm", "t7 AND t1 AND t2",
           "t5 AND t5", "t1 AND t10", "t2 AND t10", "t10 AND t3 AND t1", "t9 AND t10"]


@pytest.fixture
def cand_cost():
    old = os.environ.get("TRN_CAND_COST")
    yield lambda v: os.environ.pop("TRN_CAND_COST", None) if v is None else os.environ.__setitem__("TRN_CAND_COST", str(v))
    if old is None:
        os.environ.pop("TRN_CAND_COST", None)
    else:
        os.environ["TRN_CAND_COST"] = old


@pytest.mark.parametrize("cost", [1, None, 0], ids=["forced", "default", "off"])
def test_candidate_conjunctions_match_reference(ref, cand_cost, cost):
    cand_cost(cost)  # read by trn_create (unset: the planner's default crossover)
    p = Pair(ref, tb.CODEC_GOOGLE, make_lists(), NDOCS)
    plans = [p.plan(q) for q in QUERIES]
    res = p.gpu.exec_batch(plans, tb.MODE_DOCS_ONLY)
    routes = list(p.gpu.last_routes())
    assert routes == list(tb.debug_plan(tb.CODEC_GOOGLE, p.index, p.terms, plans, tb.MODE_DOCS_ONLY, max_docid=NDOCS)[0])
    if cost == 0:
        assert tb.ROUTE_CANDIDATE not in routes
    else:  # every all-term AND of two known terms is candidate-driven when forced; at the default crossover only the sparse leads are
        assert routes.count(tb.ROUTE_CANDIDATE) >= (17 if cost == 1 else 3), routes
    for i, q in enumerate(QUERIES):
        want, _ = p.ref.exec(q, False, NDOCS + 1)
        assert_same_docs(res.query(i)[0], want, f"[{q}] cost={cost}")
        assert int(res.match_counts[i]) == len(want)
    # masked documents are dropped before emission
    rng = np.random.default_rng(5)
    masked = np.unique(rng.integers(1, NDOCS + 1, 200_000)).astype(np.uint32)
    p.gpu.set_masked_documents(masked)
    res = p.gpu.exec_batch(plans, tb.MODE_DOCS_ONLY)
    for i, q in enumerate(QUERIES):
        want, _ = p.ref.exec_masked(q, False, masked, NDOCS + 1)
        assert_same_docs(res.query(i)[0], want, f"[{q}] masked cost={cost}")


@pytest.mark.parametrize("cost", [1, None], ids=["forced", "default"])
def test_candidate_driven_trees_match_reference(ref, cand_cost, cost):
    """every tree with 2..8 distinct terms one of which all matches must hold: lead candidates + membership probes + truth table"""
    cand_cost(cost)
    ndocs = 300_000
    p = Pair(ref, tb.CODEC_GOOGLE, closed_form_lists(ndocs), ndocs)
    qs = [(q, 0, 0) for q in TEMPLATES + EXTRA] + [(q, 8, 0) for q in OPTIONAL_QUERIES] + [(q, 16, m) for q, m in SOME_QUERIES]
    plans = [tb.parse_query(q, p.tdict, min_match=m or None) for q, _, m in qs]
    res = p.gpu.exec_batch(plans, tb.MODE_DOCS_ONLY)
    assert (list(p.gpu.last_routes()).count(tb.ROUTE_CANDIDATE) >= 20) == (cost == 1)  # (the closed-form terms are too dense for the default)
    for i, (q, flags, m) in enumerate(qs):
        want, _ = p.ref.exec(q, False, ndocs + 1, parser_flags=flags, min_match=m)
        assert_same_docs(res.query(i)[0], want, f"[{q}] min={m} cost={cost}")
