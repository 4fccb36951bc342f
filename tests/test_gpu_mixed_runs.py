"""The flat ANDs with one decoded operand on their run-major tickets (exec_docs.cuh mixed_run_exec): every result equals the reference
(oracle/_ref), and the plain and compact streams equal word for word those of the same batch on a source created with TRN_MIXED_RUNS=0
(the per-tile path).  The corpus and batch are test_mixed_runs_cpu's: leads whose tiles take the U16, U8B and bitmap forms and a full
256-docID bucket, two bitmap operands, a lead with gaps of 20 000 (3-byte codes; blocks across tiles and runs), a query of one tile,
narrow-span bitmap terms, beside all-bitmap, two-decoded, candidate-driven, flat-tree and flat-OR plans.  Also: TRN_DOCS_SHIFT 13 / 14 / 17,
masked documents, the pipelined trn_exec_batch, 2 and 3 shards, and the corpus translated to end at 2^32 - 2."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

import trinity_b200 as tb
from refharness import RefIndex
from test_gpu_emit_layout import ENC, QItems
from test_mixed_runs_cpu import FULL, LISTS, MIXED, NAMES, QUERIES, S, build
from util import assert_same_docs

pytestmark = pytest.mark.gpu

G = tb.CODEC_GOOGLE
TOP = 2**32 - 2
DELTA = TOP - S


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


def _source(index, terms, max_docid, env):
    with _env(env):
        g = tb.GpuIndexSource(0)
    g.upload(G, index, terms, max_docid)
    return g


def _streams(g, plans):
    """(plain docIDs per query, compact results decoded per query, (offsets, words, item_desc, qitems) of the compact stream, routes)"""
    plain = g.exec_batch(plans, tb.MODE_DOCS_ONLY)
    docs = [plain.query(i)[0].copy() for i in range(len(plans))]
    routes = list(g.last_routes())
    comp = g.exec_batch(plans, tb.MODE_DOCS_COMPACT, copy=False)
    assert list(g.last_routes()) == routes
    raw, nq = comp.raw, comp.nq
    off = np.ctypeslib.as_array(raw.offsets, shape=(nq + 1,)).copy()
    words = np.ctypeslib.as_array(raw.words, shape=(max(int(raw.total_words), 1),))[: int(raw.total_words)].copy()
    desc = np.ctypeslib.as_array(raw.item_desc, shape=(max(comp.nitems, 1),))[: comp.nitems].copy()
    qi = C.cast(raw.qitems, C.POINTER(QItems))
    qitems = [(qi[q].item_base, qi[q].nitems, qi[q].tile_lo, qi[q].tile_shift) for q in range(nq)]
    decoded = [comp.decode_query(i).copy() for i in range(nq)]
    return docs, decoded, (off, words, desc, qitems), routes


def _check(index, terms, max_docid, plans, want, label, env=None, masked=None):
    """runs on vs off (TRN_MIXED_RUNS) vs want, both modes; the batch must use the mixed tickets. Returns the on-source's compact stream."""
    env = dict(env or {})
    with _env(env):
        routes, _ = tb.debug_plan(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=max_docid)
        assert len(tb.debug_mixed_runs(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=max_docid)[1]), label
    out = {}
    for runs in ("1", "0"):
        g = _source(index, terms, max_docid, {**env, "TRN_MIXED_RUNS": runs})
        try:
            if masked is not None:
                g.set_masked_documents(masked)
            out[runs] = _streams(g, plans)
        finally:
            g.close()
    for runs, (docs, decoded, _, r) in out.items():
        assert r == list(routes), (label, runs)
        for i in range(len(plans)):
            assert_same_docs(docs[i], want[i], f"{label} [{i}] mixed runs {runs}, plain")
            assert_same_docs(decoded[i], want[i], f"{label} [{i}] mixed runs {runs}, compact")
    (on_off, on_words, on_desc, on_qi), (off_off, off_words, off_desc, off_qi) = out["1"][2], out["0"][2]
    assert on_qi == off_qi, label
    assert np.array_equal(on_desc, off_desc), f"{label}: item_desc differs at {np.flatnonzero(on_desc != off_desc)[:8]}"
    assert np.array_equal(on_off, off_off), f"{label}: query offsets differ"
    assert np.array_equal(on_words, off_words), f"{label}: compact words differ at {np.flatnonzero(on_words != off_words)[:8]}"
    return out["1"][2]


@pytest.fixture(scope="module")
def world(ref):
    r = RefIndex(ref, G)
    for n in NAMES:
        r.add_term(n, LISTS[n], 1 + LISTS[n] % 3)
    r.finish(S)
    tdict = tb.TermDictionary(NAMES)
    return dict(ref=r, tdict=tdict, plans=[tb.parse_query(q, tdict) for q in QUERIES])


def _want(w, shift=0):
    return [(w["ref"].exec(q, False, S + 1)[0].astype(np.uint64) + shift).astype(np.uint32) for q in QUERIES]


@pytest.mark.parametrize("docs_shift", [13, 14, 17])
def test_results_equal_reference_and_runs_off(world, docs_shift):
    index, terms = build(G)
    off, words, desc, qitems = _check(index, terms, S, world["plans"], _want(world), f"shift {docs_shift}", {"TRN_DOCS_SHIFT": str(docs_shift)})
    if docs_shift != 14:
        return
    # the mixed queries' tiles take every form, and the tile with the full bucket is not U8B
    seen = set()
    for q in (QUERIES.index(m) for m in MIXED):
        base, n, tile_lo, shift = qitems[q]
        seen |= {int(d) >> 30 for d in desc[base: base + n] if d & 0x3FFFFFFF}
    assert {ENC["u16"], ENC["u8b"], ENC["bitmap"]} <= seen, seen
    base, n, tile_lo, shift = qitems[QUERIES.index("x AND f")]
    d = int(desc[base + (int(FULL[0]) >> shift) - tile_lo])
    assert d >> 30 == ENC["u16"] and (d & 0x3FFFFFFF) < 1024, d  # U8B would be smaller, but its count byte cannot hold 256


def test_masked_documents(world):
    rng = np.random.default_rng(5)
    pool = np.unique(np.concatenate([LISTS["x"][::3], LISTS["m"][::2], LISTS["y"][::4], FULL[::9], LISTS["z"][::2]]))
    masked = np.sort(rng.choice(pool, size=len(pool) // 2, replace=False)).astype(np.uint32)
    want = [world["ref"].exec_masked(q, False, masked, S + 1)[0] for q in QUERIES]
    index, terms = build(G)
    _check(index, terms, S, world["plans"], want, "masked", masked=masked)


def test_pipelined(world):
    env = {"TRN_PIPELINE_CHUNKS": "8", "TRN_CHUNK_POSTINGS": "1", "TRN_CHUNK_RULE": "postings"}
    index, terms = build(G)
    plans = world["plans"] * 5  # >= 64 queries: split into chunks
    with _env(env):
        _check(index, terms, S, plans, _want(world) * 5, "pipelined")


@pytest.mark.parametrize("nshards", [2, 3])
def test_shards(world, nshards):
    cuts = [1] + [int(S * (i + 1) / nshards) + 1 for i in range(nshards - 1)] + [S + 1]
    want = _want(world)
    checked = 0
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        index, terms = build(G, lo=lo, hi=hi - 1)
        part = [w[(w >= lo) & (w < hi)] for w in want]
        plans = [tb.parse_query(q, world["tdict"]) for q in QUERIES]
        if len(tb.debug_mixed_runs(G, index, terms, plans, tb.MODE_DOCS_ONLY, max_docid=S)[1]):
            _check(index, terms, S, plans, part, f"shard [{lo}, {hi})")
            checked += 1
    assert checked


def test_top_of_the_docid_space(world):
    index, terms = build(G, shift=DELTA)
    plans = [tb.parse_query(q, tb.TermDictionary(NAMES)) for q in QUERIES]
    _check(index, terms, TOP, plans, _want(world, DELTA), "top")
