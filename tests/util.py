"""Shared helpers for the parity tests (test infrastructure)."""
from __future__ import annotations

import numpy as np

import trinity_b200 as tb
from refharness import RefIndex

PRIMES = [2, 3, 5, 7, 11, 13, 17, 19, 23, 29]
PRIMES18 = PRIMES + [31, 37, 41, 43, 47, 53, 59, 61]  # t11 .. t18: plans wider than the kernels' leaf limits


def closed_form_lists(ndocs: int, primes=PRIMES):
    """term t_i = multiples of primes[i] (SURVEY.md Appendix C); freq pattern gives BM25 something to chew on"""
    out = []
    for p in primes:
        d = np.arange(p, ndocs + 1, p, dtype=np.uint32)
        f = (1 + (d // p) % 5).astype(np.uint32)
        out.append((d, f))
    return out


class Pair:
    """The same postings indexed twice: through OUR host encoders (-> GPU engine) and through the REFERENCE encoders
    (-> reference exec_query).  `names[i]` is the term of lists[i]."""

    def __init__(self, ref, codec: int, lists, ndocs: int, names=None, device: int = 0, upload: bool = True):
        self.codec, self.ndocs = codec, ndocs
        self.names = names or [f"t{i + 1}" for i in range(len(lists))]
        self.lists = lists
        b = tb.IndexBuilder(codec)
        self.ref = RefIndex(ref, codec)
        for n, (d, f) in zip(self.names, lists):
            b.add_term(d, f)
            self.ref.add_term(n, d, f)
        self.ref.finish(ndocs)
        self.index, self.terms = b.index(), b.terms_array()
        self.tdict = tb.TermDictionary(self.names)
        self.gpu = None
        if upload:
            self.gpu = tb.GpuIndexSource(device)
            self.gpu.upload(codec, self.index, self.terms, ndocs)

    def plan(self, text: str, scored: bool = False):
        nodes = tb.parse_query(text, self.tdict)
        if scored:
            self.gpu.set_bm25_weights(nodes, self.ndocs)
        return nodes


def merged_topk(gpus, plans, k):
    """SCORED_TOPK on every shard, the per-shard lists gathered as [shard][nq][k] on the device and merged by trn_merge_topk
    (the exchange step of the multi-GPU path) -> per query (docIDs, scores), padding dropped"""
    import torch
    from trinity_b200.sharded import device_view
    ns, nq = len(gpus), len(plans)
    gd = torch.zeros((ns, nq, k), dtype=torch.int32, device="cuda")
    gs = torch.zeros((ns, nq, k), dtype=torch.float32, device="cuda")
    for si, g in enumerate(gpus):
        g.exec_batch_device(plans, tb.MODE_SCORED_TOPK, k)
        dptr, sptr, _ = g.last_topk_device()
        torch.cuda.synchronize()
        gd[si].view(-1).copy_(device_view(dptr, nq * k, torch.int32))
        gs[si].view(-1).copy_(device_view(sptr, nq * k, torch.float32))
    md = torch.zeros((nq, k), dtype=torch.int32, device="cuda")
    ms = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    gpus[0].merge_topk(gd.data_ptr(), gs.data_ptr(), ns, nq, k, md.data_ptr(), ms.data_ptr())
    torch.cuda.synchronize()
    md, ms = md.cpu().numpy().view(np.uint32), ms.cpu().numpy()
    return [(md[i][ms[i] >= 0], ms[i][ms[i] >= 0]) for i in range(nq)]


def assert_same_docs(got: np.ndarray, want: np.ndarray, what: str):
    if len(got) != len(want) or not np.array_equal(got, want):
        n = min(len(got), len(want))
        bad = np.flatnonzero(got[:n] != want[:n])
        first = int(bad[0]) if len(bad) else n
        lo = max(0, first - 3)
        raise AssertionError(f"{what}: docID sets differ: got {len(got)} want {len(want)}; first mismatch at #{first}: "
                             f"got {got[lo:first + 4]} want {want[lo:first + 4]}")


def assert_close_scores(got: np.ndarray, want: np.ndarray, what: str, rtol: float = 1e-5):
    """north_star tolerance: BM25 within 1e-5 relative of the reference CPU exec"""
    want = np.asarray(want, np.float64)
    got = np.asarray(got, np.float64)
    err = np.abs(got - want) / np.maximum(np.abs(want), 1e-30)
    err[(want == 0) & (got == 0)] = 0
    if err.size and err.max() > rtol:
        i = int(err.argmax())
        raise AssertionError(f"{what}: score mismatch at #{i}: got {got[i]!r} want {want[i]!r} rel {err[i]:.3e}")


def ref_topk(ids: np.ndarray, scores: np.ndarray, k: int):
    """(score desc, docID asc) top-k of the reference's full (id, score) stream"""
    order = np.lexsort((ids, -scores))[:k]
    return ids[order], scores[order]


def assert_topk_exact(gd, gs, rd, rs_all, k, what, rtol=1e-5):
    """strict top-k parity for corpora whose tie classes come out bit-identical on both sides: the docIDs equal the reference's
    (score desc, docID asc) top-k at EVERY rank, ties included, and the scores agree within rtol.  The reference's scores are ranked as
    float32, the type the top-k sink keeps (a tie class the GPU sees as one float is one class here too)."""
    rd = np.asarray(rd, np.uint32)
    rs32 = np.asarray(rs_all, np.float32)
    order = np.lexsort((rd, -rs32))[:k]
    td, ts = rd[order], np.asarray(rs_all, np.float64)[order]
    gd = np.asarray(gd, np.uint32)
    assert len(gd) == len(td), f"{what}: top-k length {len(gd)} != {len(td)}"
    if not np.array_equal(gd, td):
        i = int(np.flatnonzero(gd != td)[0])
        lo = max(0, i - 2)
        raise AssertionError(f"{what}: top-k docID at rank {i}: got {gd[lo:i + 3]} (scores {np.asarray(gs)[lo:i + 3]}) "
                             f"want {td[lo:i + 3]} (scores {ts[lo:i + 3]})")
    assert_close_scores(gs, ts, what + " (top-k scores)", rtol)


def assert_topk_equal(gd, gs, rd, rs_all, k, what, rtol=1e-5):
    """top-k parity modulo ties at the cut (SURVEY.md 8d): scores must agree position by position within rtol;
    docIDs must agree wherever the reference score is separated from its neighbours by more than the tolerance."""
    td, ts = ref_topk(rd, rs_all, k)
    assert len(gd) == len(td), f"{what}: top-k length {len(gd)} != {len(td)}"
    assert_close_scores(gs, ts, what + " (top-k scores)", rtol)
    full_sorted = np.sort(rs_all)[::-1]
    for i in range(len(td)):
        s = ts[i]
        tol = abs(s) * 4 * rtol + 1e-12
        near = np.count_nonzero(np.abs(full_sorted - s) <= tol)
        if near == 1:
            assert gd[i] == td[i], f"{what}: top-k docID at rank {i}: got {gd[i]} want {td[i]} (score {s})"
    # every returned doc must really have (approximately) the score we report
    lookup = dict(zip(rd.tolist(), rs_all.tolist()))
    for d, s in zip(gd.tolist(), gs.tolist()):
        assert d in lookup, f"{what}: top-k returned a non-matching doc {d}"
        assert abs(lookup[d] - s) <= abs(lookup[d]) * rtol + 1e-12, f"{what}: doc {d} score {s} vs reference {lookup[d]}"
