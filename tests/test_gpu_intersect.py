"""Query-token intersections on the device (GpuIndexSource.intersect / trn_intersect) against the reference's own intersect() on both
codecs: a single source as a {mask: count} dict (the reference leaves ties of its order undefined), the collection form exactly.  The
device order is checked against finalize()'s, refined by mask."""
import os
import random

import numpy as np
import pytest

import trinity_b200 as tb
from isectutil import RefIsect, considered_stream, consider_sequential, finalize_order
from trinity_b200.segments import SegmentCollection

pytestmark = pytest.mark.gpu
CODECS = pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])


@pytest.fixture(scope="module")
def risect():
    return RefIsect()


class Src:
    """the same postings as a device source and as a reference source (the host encoder writes the reference's bytes)"""

    def __init__(self, risect, codec, lists, max_docid, masked=()):
        self.names = list(lists)
        b = tb.IndexBuilder(codec)
        for n in self.names:
            d = np.asarray(lists[n], np.uint32)
            b.add_term(d, np.ones(len(d), np.uint32))
        self.index, self.terms, self.hits = b.index(), b.terms_array(), b.hits()
        self.ref = risect.source(codec, self.index, self.names, self.terms, self.hits)
        self.gpu = tb.GpuIndexSource(0)
        self.gpu.upload(codec, self.index, self.terms, max_docid)
        self.masked = list(masked)
        if self.masked:
            self.gpu.set_masked_documents(self.masked)
        self.tdict = tb.TermDictionary(self.names)

    def ids(self, tok):
        return [[self.tdict.term_id(t) for t in g] for g in tok]

    def check(self, tok, got=None):
        want = self.ref.intersect(tok, self.masked)
        if got is None:
            got = self.gpu.intersect(self.ids(tok))
        assert dict(got) == dict(want), tok
        assert len(got) == len(dict(got))
        assert got == finalize_order(got)
        return got


def random_lists(seed, nterms, ndocs):
    rng = np.random.default_rng(seed)
    out = {}
    for i in range(nterms):
        df = int(rng.integers(1, max(2, ndocs // (i + 2))))
        out[f"k{i}"] = np.sort(rng.choice(np.arange(1, ndocs), size=df, replace=False))
    out["empty"] = np.zeros(0, np.uint32)
    return out


def random_request(rng, names, maxg=8):
    ng = rng.randint(1, maxg)
    tok = [rng.sample(names, rng.randint(1, 3)) for _ in range(ng)]
    r = rng.random()
    if r < 0.15:
        tok[rng.randrange(ng)].append("nosuchtoken")  # unknown: origMask = 0
    elif r < 0.25:
        tok[rng.randrange(ng)].append("empty")  # a 0-document term is unknown too
    elif r < 0.35 and ng > 1:
        tok[1].append(tok[0][0])  # one token in two groups
    return tok


@CODECS
def test_random_requests_and_batch(risect, codec):
    s = Src(risect, codec, random_lists(5, 12, 40_000), 40_000, masked=range(7, 40_000, 13))
    rng = random.Random(11)
    names = [n for n in s.names if n != "empty"]
    reqs = [random_request(rng, names) for _ in range(220)]
    reqs += [[["nosuch"], ["other"]], [["empty"]], []]  # all tokens unknown / no group: empty
    res = s.gpu.intersect_batch([s.ids(t) for t in reqs])
    assert res.postings > 0 and res.distinct > 0
    for i, t in enumerate(reqs):
        s.check(t, res[i])
    for i in (0, 17, 101, 219):  # a request alone equals it in the batch
        assert s.gpu.intersect(s.ids(reqs[i])) == res[i]
    assert res[-1] == [] and res[-2] == [] and res[-3] == []


def stream_lists(stream, ngroups):
    """one term g<i> per group: the documents whose mask holds bit i"""
    return {f"g{g}": [d for d, m in stream if (m >> g) & 1] for g in range(ngroups)}


def stream_of(seq, start=1, gap=1):
    out, d = [], start
    for m in seq:
        out.append((d, m))
        d += gap
    return out


QUIRKS = {
    # a run of 0b01 absorbed by the earlier strict superset 0b11: L - 1
    "absorbed_run": ([0b011, 0b001, 0b001, 0b001, 0b100], 3),
    # 0b01 seen (and counted) before its superset: its count is lost when 0b11 removes it
    "subset_before_superset": ([0b001, 0b001, 0b011, 0b001, 0b001, 0b100], 3),
    # two maximal supersets of 0b001; the swap-removal order decides which one a later 0b001 run counts on
    "swap_order": ([0b001, 0b100, 0b011, 0b110, 0b101, 0b001, 0b001, 0b010, 0b010], 3),
    # a run continued across a document of the whole query (origMask, not considered) and across a masked document
    "run_across_orig_and_masked": ([0b01, 0b01, 0b11, 0b01, 0b10, 0b01, 0b01, 0b01], 2),
}


@CODECS
@pytest.mark.parametrize("name", list(QUIRKS))
def test_crafted_quirks(risect, codec, name):
    seq, ng = QUIRKS[name]
    stream = stream_of(seq, start=100, gap=3)
    masked = [stream[6][0]] if name == "run_across_orig_and_masked" else []
    s = Src(risect, codec, stream_lists(stream, ng), 10_000, masked)
    tok = [[f"g{g}"] for g in range(ng)]
    got = s.check(tok)
    gd = [[d for d, m in stream if (m >> g) & 1] for g in range(ng)]
    assert dict(got) == consider_sequential([m for _, m in considered_stream(gd, masked)])


@CODECS
@pytest.mark.parametrize("ngroups", [3, 12, 24, 64])
def test_runs_across_tile_edges(risect, codec, ngroups):
    """every tile size the kernels use (2^13 documents up to 8 groups, 2^12, 2^11, 2^10 for 64): runs of equal masks straddle the edges,
    with masks that change between edges; 64 groups set bit 63"""
    lg = max(3, (ngroups - 1).bit_length())
    W = 1 << (16 - lg)
    rng = random.Random(ngroups)
    stream, prev = [], 0
    for k in range(1, 9):
        m = rng.getrandbits(ngroups) or 1
        if k % 3 == 0:
            m = prev  # the same mask on both sides of an edge, across tiles without a considered document in between
        for d in range(k * 3 * W - 3, k * 3 * W + 3):
            stream.append((d, m))
        prev = m
    stream.append((40 * W, 1 << (ngroups - 1)))
    s = Src(risect, codec, stream_lists(stream, ngroups), 41 * W)
    tok = [[f"g{g}"] for g in range(ngroups)]
    got = s.check(tok)
    assert any(m >> (ngroups - 1) for m, _ in got)


def test_dense_bitmaps_and_without(risect):
    n = 400_000
    lists = {"dense": np.arange(1, n, 2), "mid": np.arange(3, n, 7), "rare": np.arange(5, n, 997), "other": np.arange(2, n, 3)}
    reqs = [[["dense"], ["mid"]], [["dense", "other"], ["rare"], ["mid"]], [["dense"], ["dense", "rare"]], [["mid"], ["nosuch"], ["dense"]]]
    results = []
    for env in (None, "0"):
        old = os.environ.get("TRN_DENSE_BITMAPS")
        if env is not None:
            os.environ["TRN_DENSE_BITMAPS"] = env
        try:
            s = Src(risect, tb.CODEC_GOOGLE, lists, n, masked=range(11, n, 101))
        finally:
            if old is None:
                os.environ.pop("TRN_DENSE_BITMAPS", None)
            else:
                os.environ["TRN_DENSE_BITMAPS"] = old
        assert (s.gpu.info()["dense_terms"] > 0) == (env is None)
        res = s.gpu.intersect_batch([s.ids(t) for t in reqs])
        for i, t in enumerate(reqs):
            s.check(t, res[i])
        results.append(res.results)
    assert results[0] == results[1]


@CODECS
def test_top_of_docid_space(risect, codec):
    """by translation: the device source holds the reference corpus shifted so that its largest docID is 2^32 - 2"""
    S = 300_000
    top = 2**32 - 2
    delta = top - S
    rng = np.random.default_rng(3)
    lists = {f"k{i}": np.unique(np.concatenate([np.sort(rng.choice(np.arange(1, S), size=S // (3 + 5 * i), replace=False)), [S - i, S]])) for i in range(5)}
    masked = list(range(S - 400, S, 9))
    ref = Src(risect, codec, lists, S, masked)
    b = tb.IndexBuilder(codec)
    for n in lists:
        b.add_term(np.asarray(lists[n], np.uint64) + delta, np.ones(len(lists[n]), np.uint32))
    g = tb.GpuIndexSource(0)
    g.upload(codec, b.index(), b.terms_array(), top)
    g.set_masked_documents(np.asarray(masked, np.uint64) + delta)
    rng2 = random.Random(2)
    for _ in range(12):
        tok = random_request(rng2, list(lists), 5)
        ref.check(tok, g.intersect(ref.ids(tok)))


@CODECS
def test_segment_collection_three_generations(risect, codec, tmp_path, ref):
    def lists(seed, lo, hi):
        rng = np.random.default_rng(seed)
        out = {}
        for t in range(1, 7):
            df = max(1, (hi - lo) // (t + 1))
            out[f"w{t}"] = (np.sort(rng.choice(np.arange(lo, hi), size=df, replace=False)).astype(np.uint32), np.ones(df, np.uint32))
        return out

    dirs = [tmp_path / "1", tmp_path / "2", tmp_path / "3"]
    for d in dirs:
        d.mkdir()
    ref.segment_write(codec, dirs[0], lists(1, 1, 60_000))
    ref.segment_write(codec, dirs[1], lists(2, 40_000, 90_000), np.arange(3, 20_000, 11, dtype=np.uint32), replace_below=60_000)
    ref.segment_write(codec, dirs[2], lists(3, 70_000, 120_000), np.arange(45_000, 50_000, 3, dtype=np.uint32), replace_below=90_000)
    col = SegmentCollection(dirs)
    rcol = risect.collection(sorted(dirs, key=lambda p: -int(p.name)))
    for tok in ([["w1"], ["w2"], ["w3"]], [["w1", "w4"], ["w2"], ["nosuch"]], [["w5"], ["w6"], ["w1"], ["w2", "w3"]], [["w2"]]):
        assert col.intersect(tok) == rcol.intersect_collection(tok), tok


def test_refusals_and_limits(risect):
    lists = {f"k{i}": np.arange(1 + i, 5000, 2 + i % 7) for i in range(70)}
    s = Src(risect, tb.CODEC_GOOGLE, lists, 5000)
    ids = list(range(70))
    s.gpu.intersect([[t] for t in ids[:64]])
    with pytest.raises(tb.TrinityError, match="rc=-1"):
        s.gpu.intersect([[t] for t in ids[:65]])
    s.gpu.intersect([ids[:64]] * 8)  # 512 known tokens (a token in several groups counts in each)
    with pytest.raises(tb.TrinityError, match="rc=-1"):
        s.gpu.intersect([ids[:64]] * 8 + [[ids[0]]])
    with pytest.raises(tb.TrinityError, match="rc=-7"):
        s.gpu.intersect([[0], [1]], stopwords_mask=1)
    s.check([[f"k{i}"] for i in range(64)])


def test_mask_limit(risect, monkeypatch):
    lists = {f"k{i}": np.arange(1 + i, 20_000, 3 + i) for i in range(10)}
    probe = Src(risect, tb.CODEC_GOOGLE, lists, 20_000)
    tok = [[f"k{i}"] for i in range(10)]
    res = probe.gpu.intersect_batch([probe.ids(tok)])
    d = res.distinct
    assert d > 50
    for cap, ok in ((d, True), (d - 1, False)):
        monkeypatch.setenv("TRN_ISECT_MAX_MASKS", str(cap))
        s = Src(risect, tb.CODEC_GOOGLE, lists, 20_000)
        if ok:
            s.check(tok)
        else:
            with pytest.raises(tb.TrinityError, match="rc=-6.*request 1"):
                s.gpu.intersect_batch([[[0]], s.ids(tok)])
