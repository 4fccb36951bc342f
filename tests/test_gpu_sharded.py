"""The docID-sharded (multi-GPU) path checked on ONE GPU against the UNSHARDED reference: S doc_range shards of the same index are
uploaded into S separate device-resident IndexSources (what S ranks would hold), every shard runs the batch, DocumentsOnly results
concatenate in shard order, top-k lists go through the exchange step's own merge kernel (`trn_merge_topk` == k_topk_merge on the
all-gathered [shard][nq][k] layout).  Reference: exec_query over the whole index (exec.h:56-61,84-177; BM25 over collection statistics,
similarity.h:209-217).  Covers shards whose first docID is not 1, shards where a term is empty, k that no shard can fill, ties across
shards.  The closed-form freq pattern gives exact ties wherever a document's score has at most two contributions (a + b is the same float
in either order): those top-k plans are checked strictly, docID order at every rank included (assert_topk_exact).  The 10-term OR and the
two-conjunction OR sum more contributions, in an order that differs between the kernels and the reference, so their tie classes need not
be bit-identical: they are checked modulo near-ties (assert_topk_equal)."""
import numpy as np
import pytest
import torch

import trinity_b200 as tb
from refharness import RefIndex
from trinity_b200.sharded import device_view, shard_range
from util import Pair, assert_same_docs, assert_topk_equal, assert_topk_exact, closed_form_lists

pytestmark = pytest.mark.gpu
CODECS = [tb.CODEC_GOOGLE, tb.CODEC_LUCENE]

DOCS_QUERIES = [
    "t1 AND t2", "t3 OR t7 OR t9", "t1 AND (t2 OR t3) NOT t5", "(t1 AND t2) OR (t3 AND t4) OR (t5 AND t6) NOT t7 NOT t8",
    "t10", "t9 AND t10", "rare AND t1", "rare OR t10", "t2 AND t3 AND t5 NOT rare", "[t1, t2, t3, t4]",
]
TOPK_QUERIES = [" OR ".join(f"t{i}" for i in range(1, 11)), "t1 AND t2", "t3 OR t7", "rare OR t10", "t10", "rare", "(t1 AND t2) OR (t3 AND t4)"]
EXACT_TIES = {"t1 AND t2", "t3 OR t7", "rare OR t10", "t10", "rare"}  # at most two contributions per document


def _lists(ndocs):
    """closed-form multiples-of-primes lists (identical freq patterns => score ties within and ACROSS shards) + one rare term that
    lives in a single shard (empty term everywhere else)"""
    lists = closed_form_lists(ndocs)
    rare = np.array([ndocs // 2 + 7, ndocs // 2 + 4099, ndocs // 2 + 5000], np.uint32)
    lists.append((rare, np.array([3, 1, 2], np.uint32)))
    names = [f"t{i + 1}" for i in range(10)] + ["rare"]
    return lists, names


class Shard:
    def __init__(self, codec, lists, names, lo, hi, ndocs, full_df):
        b = tb.IndexBuilder(codec)
        for d, f in lists:
            keep = (d >= lo) & (d <= hi)
            b.add_term(d[keep], f[keep])
        self.gpu = tb.GpuIndexSource(0)
        self.gpu.upload(codec, b.index(), b.terms_array(), ndocs)
        self.tdict = tb.TermDictionary(names)
        self.full_df, self.ndocs = full_df, ndocs

    def plan(self, text, scored=False, min_match=None):
        nodes = tb.parse_query(text, self.tdict, min_match=min_match)
        if scored:  # GLOBAL document frequencies: every shard scores like the unsharded collection (similarity.h:209-217)
            for x in nodes:
                if x["kind"] == tb.NODE_TERM and x["term"] != tb.EMPTY_TERM:
                    x["weight"] = tb.bm25_idf(int(self.full_df[x["term"]]), self.ndocs)
        return nodes


@pytest.mark.parametrize("codec", CODECS, ids=["google", "lucene"])
@pytest.mark.parametrize("nshards", [2, 3, 8])
def test_sharded_results_equal_unsharded_reference(ref, codec, nshards):
    ndocs = 400_000
    lists, names = _lists(ndocs)
    whole = Pair(ref, codec, lists, ndocs, names=names, upload=False)
    full_df = np.array([len(d) for d, _ in lists])
    shards = [Shard(codec, lists, names, *shard_range(ndocs, r, nshards), ndocs, full_df) for r in range(nshards)]

    # ---- DocumentsOnly: shard order == docID order
    mm = {q: (2 if q.startswith("[") else None) for q in DOCS_QUERIES}
    parts = [s.gpu.exec_batch([s.plan(q, min_match=mm[q]) for q in DOCS_QUERIES], tb.MODE_DOCS_ONLY) for s in shards]
    for i, q in enumerate(DOCS_QUERIES):
        want, _ = whole.ref.exec(q, False, ndocs + 1, parser_flags=16 if q.startswith("[") else 0, min_match=mm[q] or 0)
        got = np.concatenate([p.query(i)[0] for p in parts])
        assert_same_docs(got, want, f"{nshards} shards [{q}]")
        assert sum(int(p.match_counts[i]) for p in parts) == len(want)

    # ---- top-k: per-shard lists -> [shard][nq][k] (what the all-gather delivers) -> trn_merge_topk
    nq = len(TOPK_QUERIES)
    for k in (7, 100):  # 100: no shard of the rare-term queries can fill k; 7: does not divide anything evenly
        gd = torch.zeros((nshards, nq, k), dtype=torch.int32, device="cuda")
        gs = torch.zeros((nshards, nq, k), dtype=torch.float32, device="cuda")
        counts = np.zeros(nq, np.int64)
        for si, s in enumerate(shards):
            s.gpu.exec_batch_device([s.plan(q, scored=True) for q in TOPK_QUERIES], tb.MODE_SCORED_TOPK, k)
            dptr, sptr, _ = s.gpu.last_topk_device()
            torch.cuda.synchronize()
            gd[si].view(-1).copy_(device_view(dptr, nq * k, torch.int32))
            gs[si].view(-1).copy_(device_view(sptr, nq * k, torch.float32))
            counts += np.asarray(s.gpu.fetch().match_counts, np.int64)
        md = torch.zeros((nq, k), dtype=torch.int32, device="cuda")
        ms = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        shards[0].gpu.merge_topk(gd.data_ptr(), gs.data_ptr(), nshards, nq, k, md.data_ptr(), ms.data_ptr())
        torch.cuda.synchronize()
        md, ms = md.cpu().numpy().view(np.uint32), ms.cpu().numpy()
        for i, q in enumerate(TOPK_QUERIES):
            wd, ws = whole.ref.exec(q, True, ndocs + 1)
            assert counts[i] == len(wd), f"{nshards} shards [{q}]: summed match counts"
            keep = ms[i] >= 0
            check = assert_topk_exact if q in EXACT_TIES else assert_topk_equal
            check(md[i][keep], ms[i][keep], wd, ws, k, f"{nshards} shards [{q}] k={k}")
    for s in shards:
        s.gpu.close()


def test_sharded_synthetic_index_equals_unsharded_reference(ref):
    """the bench's own index family (Zipfian SynthIndex, doc_range shards incl. uneven ones) on the headline query shapes"""
    from bench import gen_queries
    ndocs, nterms, min_df, k = 3_000_000, 96, 40, 100
    full = tb.SynthIndex(tb.CODEC_GOOGLE, ndocs, nterms, min_df=min_df, threads=8)
    r = RefIndex.from_bytes(ref, tb.CODEC_GOOGLE, np.asarray(full.index), np.asarray(full.hits), full.names, np.asarray(full.terms), ndocs, full.sum_hits)
    tdict = tb.TermDictionary(full.names)
    texts = gen_queries("and2", 40, nterms)[0] + gen_queries("tree8", 40, nterms)[0]
    plans = [tb.parse_query(t, tdict) for t in texts]
    ortexts = gen_queries("or10", 12, nterms)[0]
    full_df = np.asarray(full.terms["documents"])
    for nshards in (2, 5, 8):
        shards = []
        for rank in range(nshards):
            lo, hi = shard_range(ndocs, rank, nshards)
            s = tb.SynthIndex(tb.CODEC_GOOGLE, ndocs, nterms, min_df=min_df, threads=8, doc_range=(lo, hi))
            g = tb.GpuIndexSource(0)
            g.upload(tb.CODEC_GOOGLE, np.asarray(s.index), np.asarray(s.terms), ndocs)
            shards.append(g)
        parts = [g.exec_batch(plans, tb.MODE_DOCS_ONLY) for g in shards]
        for i, t in enumerate(texts):
            want, _ = r.exec(t, False, ndocs + 1)
            assert_same_docs(np.concatenate([p.query(i)[0] for p in parts]), want, f"{nshards} shards [{t}]")
        oplans = []
        for t in ortexts:
            nodes = tb.parse_query(t, tdict)
            for x in nodes:
                if x["kind"] == tb.NODE_TERM and x["term"] != tb.EMPTY_TERM:
                    x["weight"] = tb.bm25_idf(int(full_df[x["term"]]), ndocs)
            oplans.append(nodes)
        nq = len(oplans)
        gd = torch.zeros((nshards, nq, k), dtype=torch.int32, device="cuda")
        gs = torch.zeros((nshards, nq, k), dtype=torch.float32, device="cuda")
        for si, g in enumerate(shards):
            g.exec_batch_device(oplans, tb.MODE_SCORED_TOPK, k)
            dptr, sptr, _ = g.last_topk_device()
            torch.cuda.synchronize()
            gd[si].view(-1).copy_(device_view(dptr, nq * k, torch.int32))
            gs[si].view(-1).copy_(device_view(sptr, nq * k, torch.float32))
        md = torch.zeros((nq, k), dtype=torch.int32, device="cuda")
        ms = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        shards[0].merge_topk(gd.data_ptr(), gs.data_ptr(), nshards, nq, k, md.data_ptr(), ms.data_ptr())
        torch.cuda.synchronize()
        md, ms = md.cpu().numpy().view(np.uint32), ms.cpu().numpy()
        for i, t in enumerate(ortexts):
            wd, ws = r.exec(t, True, ndocs + 1)
            keep = ms[i] >= 0
            assert_topk_equal(md[i][keep], ms[i][keep], wd, ws, k, f"{nshards} shards [{t}]")
        for g in shards:
            g.close()
