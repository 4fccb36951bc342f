"""The probe bitmaps (select_probe_terms) on the device: the candidate-driven conjunction probes a term of the tier with one word load
where it would otherwise search the term's block directory.  The corpora of test_gpu_candidate_edges run at TRN_CAND_COST=1 with the
tier at its default, off (TRN_PROBE_BITMAPS=0: every term without a dense bitmap probed through its directory), over every qualifying
term, and at a budget that gives only part of the tier a bitmap, so that one query probes both ways.  Every setting's docID streams
equal the reference's (or the plain evaluator's above its docID range) and each other's; also with masked documents, per-query
document filters (the filtered instantiation), a shard that does not start at docID 1 and one that ends at the top of the docID space.
info(): the dense tier is what it was, and the probe tier's bytes are the sum of its terms' spans."""
import numpy as np
import pytest

import candutil as cu
import trinity_b200 as tb
from test_gpu_candidate_edges import Corpus, _env
from util import assert_same_docs

pytestmark = pytest.mark.gpu
G = cu.G
NONE = tb.DENSE_NONE
ALIGN = 1 << 17
OFF = {"TRN_PROBE_BITMAPS": "0"}
WIDE = {"TRN_PROBE_RATIO": "1e9", "TRN_PROBE_BUDGET": "1e9"}


@pytest.fixture
def source():
    made = []

    def make(c, env):
        with _env(env):
            g = tb.GpuIndexSource(0)
        g.upload(G, c["index"], c["terms"], c["max_docid"])
        made.append(g)
        return g

    yield make
    for g in made:
        g.close()


def _selection(c, env):
    with _env(env):
        return tb.debug_probe_terms(G, c["index"], c["terms"])


def _settings(c):
    """{name: env}: default, off, every qualifying term, and a budget that holds the densest half of those"""
    off, n, _ = _selection(c, WIDE)
    _, dense_bytes = tb.debug_dense_terms(G, c["index"], c["terms"])
    tier = np.sort(off[(off != NONE) & (off >= dense_bytes // 4)])
    half = (int(tier[n // 2]) - dense_bytes // 4) * 4 if n >= 2 else 0
    return {"default": {}, "off": OFF, "wide": WIDE, "part": {**WIDE, "TRN_PROBE_BUDGET": repr((half + 0.5) / c["index"].size)}}


def _mixes(c, plans, probe_off):
    """queries whose probed terms include one with a bitmap of either tier and one without any"""
    out = []
    for i, p in enumerate(plans):
        probed = cu.probe_order(p, c["terms"])[0][1:]
        kinds = {probe_off[t] != NONE for t in probed}
        if kinds == {True, False}:
            out.append(i)
    return out


def check_tiers(source, c, queries, routes, env=None, masked=None, filters=None, want=None, label=""):
    """the batch under every tier setting (routes as given): each stream equal to want; returns the queries that mixed probe kinds
    at the partial budget"""
    env = {"TRN_CAND_COST": "1"} if env is None else env
    plans = cu.parse(queries, c["tdict"])
    want = want if want is not None else c.want(queries, plans, masked)
    info = {}
    mixed = []
    for name, tier in _settings(c).items():
        e = {**env, **tier}
        g = source(c, e)
        if masked is not None:
            g.set_masked_documents(masked)
        f = None if filters is None else [None if x is None else tb.DocFilter(*(None if s is None else g.docset(s) for s in x)) for x in filters]
        res = g.exec_batch(plans, tb.MODE_DOCS_ONLY, filters=f)
        assert list(g.last_routes()) == list(routes), (label, name)
        for i, (q, _, m) in enumerate(queries):
            assert_same_docs(res.query(i)[0], want[i], f"{label} {name} [{q}]")
        info[name] = g.info()
        probe_off, n, nbytes = _selection(c, e)
        assert info[name]["probe_terms"] == n and info[name]["probe_bitmap_bytes"] == nbytes, (label, name)
        assert nbytes == 4 * sum(cu_span_words(c, t) for t in np.flatnonzero(probe_off != NONE) if probe_off[t] * 4 >= info[name]["dense_bitmap_bytes"])
        if name == "part":
            mixed = _mixes(c, plans, probe_off)
    assert info["off"]["probe_terms"] == 0 and info["wide"]["probe_terms"] > 0, label
    assert len({(i["dense_terms"], i["dense_bitmap_bytes"]) for i in info.values()}) == 1, label
    return mixed


def cu_span_words(c, t):
    d = c["lists"][c["names"][t]]
    return ((int(d[-1]) // ALIGN + 1) * ALIGN - int(d[0]) // ALIGN * ALIGN) // 32


def test_lead_decoder(source, ref):
    c = Corpus(cu.lead_corpus(), ref)
    qs = cu.lead_queries()
    check_tiers(source, c, qs, [tb.ROUTE_CANDIDATE] * len(qs), label="A")


def test_probes(source, ref):
    c = Corpus(cu.probe_corpus(), ref)
    qs = cu.PROBE_QUERIES
    check_tiers(source, c, qs, [tb.ROUTE_CANDIDATE] * len(qs), label="B")


def test_truth_tables_mix_probe_kinds(source, ref):
    c = Corpus(cu.truth_corpus(), ref)
    qs = cu.all_truth_queries()
    mixed = check_tiers(source, c, qs, [tb.ROUTE_CANDIDATE] * len(qs), label="C")
    assert len(mixed) > 0  # at the partial budget some queries probe one term in a bitmap and another through its directory


def test_groups_masked_and_filtered(source, ref):
    c = Corpus(cu.group_corpus(), ref)
    qs = [(q, 0, 0) for q in cu.GROUP_ROUTES]
    routes = list(cu.GROUP_ROUTES.values())
    check_tiers(source, c, qs, routes, env={}, label="D")
    rng = np.random.default_rng(23)
    g_ = np.asarray(c["lists"]["g"], np.uint32)
    masked = np.unique(np.concatenate([rng.choice(g_, 900, replace=False), rng.choice(np.arange(2, 400_001, 2, dtype=np.uint32), 5000, replace=False)]))
    check_tiers(source, c, qs, routes, env={}, masked=masked.astype(np.uint32), label="D masked")
    # per-query document filters: the filtered instantiation of the candidate-driven conjunction
    allow = np.unique(rng.choice(np.arange(1, 400_001, dtype=np.uint32), 150_000, replace=False)).astype(np.uint32)
    deny = np.unique(rng.choice(g_, 1500, replace=False)).astype(np.uint32)
    sets = [(allow, None), (None, deny), (allow, deny), None, (allow, None), (None, deny), (allow, deny)][: len(qs)]
    plans = cu.parse(qs, c["tdict"])
    want = []
    for w, s in zip(c.want(qs, plans), sets):
        w = np.asarray(w, np.uint32)
        if s is not None and s[0] is not None:
            w = w[np.isin(w, s[0])]
        if s is not None and s[1] is not None:
            w = w[~np.isin(w, s[1])]
        want.append(w)
    check_tiers(source, c, qs, routes, env={}, filters=sets, want=want, label="D filtered")


def _shifted(lists, delta):
    return {k: (np.asarray(v, np.uint64) + delta).astype(np.uint32) for k, v in lists.items()}


def test_shard_not_starting_at_one(source):
    c = Corpus(_shifted(cu.group_corpus(), 40 * ALIGN))  # whole 2^17 runs: every span keeps its size, every route its choice
    qs = [(q, 0, 0) for q in cu.GROUP_ROUTES]
    check_tiers(source, c, qs, list(cu.GROUP_ROUTES.values()), env={}, label="D shifted")


def test_top_of_the_docid_space(source):
    """the probe corpus translated so that its last docID is 2^32 - 2, and the corpus that ends there by construction"""
    lists = cu.probe_corpus()
    top = max(int(v[-1]) for v in lists.values())
    c = Corpus(_shifted(lists, cu.TOP - top))
    assert c["max_docid"] == cu.TOP
    qs = cu.PROBE_QUERIES
    check_tiers(source, c, qs, [tb.ROUTE_CANDIDATE] * len(qs), label="B at the top")
    c = Corpus(cu.top_corpus())
    qs = cu.TOP_QUERIES
    check_tiers(source, c, qs, [tb.ROUTE_CANDIDATE] * len(qs), label="F")
