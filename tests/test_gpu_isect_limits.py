"""Query-token intersections on the device at their internal switch points, on both sides, against the reference's own intersect() and
finalize()'s order: the uint8_t indexPrev past 256 antichain entries, the largest accepted request (64 groups, 512 known tokens), every
change of tile width (8/9, 16/17, 32/33 groups), and the distinct-mask table at its real limit of 65 536 and when the documents bound it."""
import random

import numpy as np
import pytest

import trinity_b200 as tb
from isectutil import RefIsect, considered_stream, consider_sequential, finalize_order
from test_gpu_intersect import Src, stream_lists

pytestmark = pytest.mark.gpu
CODECS = pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
MAX_MASKS = 1 << 16  # kIsectMaxMasks


@pytest.fixture(scope="module")
def risect():
    return RefIsect()


def tile_width(ngroups):
    """docIDs of one tile (isect_tile_shift): 2^13 up to 8 groups, halved each time the groups pass a power of two"""
    return 1 << (16 - max(3, (ngroups - 1).bit_length()))


def wide_antichain(masked_and_orig):
    """the stream of test_epoch_restatement_wide_antichain: 435 incomparable two-bit masks over 30 groups in runs of 1..4 (the antichain
    never drops an entry, so the k-th mask is entry k, and a run continued on entry k >= 256 adds to entry k & 255), then the first 100
    again (runs on entries 0..99), then two single-bit masks that earlier entries absorb.  masked_and_orig: from entry 256 on, a document
    of the whole query (origMask, not considered) or a masked document of another mask stands between the documents of a run.
    -> (stream [(docID, mask)], masked docIDs, the entry of every run such a document breaks)"""
    rng = random.Random(7)
    pairs = [(1 << a) | (1 << b) for a in range(30) for b in range(a + 1, 30)]
    rng.shuffle(pairs)
    entry = {m: k for k, m in enumerate(pairs)}
    full = (1 << 30) - 1
    s, masked, broken, d = [], [], [], 0
    for k, m in enumerate(pairs + pairs[:100] + [1 << 3, 1 << 7]):
        for r in range(rng.randint(1, 4)):
            if masked_and_orig and k >= 256 and r:
                d += 1
                if rng.random() < 0.5:
                    s.append((d, full))
                else:
                    s.append((d, pairs[rng.randrange(len(pairs))]))
                    masked.append(d)
                broken.append(entry.get(m, -1))
            d += 1
            s.append((d, m))
    return s, masked, broken


@CODECS
@pytest.mark.parametrize("variant", ["runs", "masked-and-orig"])
def test_wide_antichain_wraps_index_prev(risect, codec, variant):
    stream, masked, broken = wide_antichain(variant != "runs")
    ng = 30
    s = Src(risect, codec, stream_lists(stream, ng), stream[-1][0] + 1, masked)
    tok = [[f"g{g}"] for g in range(ng)]
    res = s.gpu.intersect_batch([s.ids(tok)])
    got = s.check(tok, res[0])
    gd = [[d for d, m in stream if (m >> g) & 1] for g in range(ng)]
    cons = [m for _, m in considered_stream(gd, masked)]
    want = consider_sequential(cons)
    assert dict(got) == want and len(got) == 435
    assert res.distinct == len(set(cons)) == 437
    assert consider_sequential(cons, index_wrap=None) != want  # the case reaches the wrap: an index that does not wrap answers otherwise
    if variant != "runs":
        assert len(masked) > 20 and len(cons) < len(stream) - len(masked)  # origMask documents stood in runs too
        assert sum(e > 255 for e in broken) > 100  # runs broken on entries whose index wraps


@CODECS
def test_largest_accepted_request(risect, codec):
    """64 groups of 8 known tokens each (512, a token in several groups counting in each), checked against the reference; one group or one
    token more is refused and the context answers again"""
    lists = {f"k{i}": np.arange(1 + i, 6000, 2 + i % 7) for i in range(70)}
    s = Src(risect, codec, lists, 6000, masked=range(5, 6000, 97))
    tok = [[f"k{(g * 8 + j) % 70}" for j in range(8)] for g in range(64)]
    res = s.gpu.intersect_batch([s.ids(tok)])
    got = s.check(tok, res[0])
    assert any(m >> 63 for m, _ in got) and res.distinct > 64
    with pytest.raises(tb.TrinityError, match="rc=-1: .*request 0: 65 token groups"):
        s.gpu.intersect(s.ids(tok + [["k0"]]))
    with pytest.raises(tb.TrinityError, match="rc=-1: .*request 0: 513 known tokens"):
        s.gpu.intersect(s.ids(tok[:63] + [tok[63] + ["k69"]]))
    assert s.gpu.intersect(s.ids(tok)) == got


@CODECS
@pytest.mark.parametrize("ngroups", [8, 9, 16, 17, 32, 33])
def test_runs_across_tile_edges_at_each_width_switch(risect, codec, ngroups):
    """both sides of each tile-width switch (2^13 | 2^12 | 2^11 | 2^10 documents): runs of equal masks straddle the edges of this width,
    a mask carried across edges with no considered document between, and the top group's bit"""
    W = tile_width(ngroups)
    assert W == {8: 1 << 13, 9: 1 << 12, 16: 1 << 12, 17: 1 << 11, 32: 1 << 11, 33: 1 << 10}[ngroups]
    rng = random.Random(100 + ngroups)
    stream, prev = [], 0
    for k in range(1, 11):
        m = rng.getrandbits(ngroups) or 1
        if k % 3 == 0:
            m = prev
        for d in range(k * 3 * W - 5, k * 3 * W + 4):
            stream.append((d, m))
        if k % 2:
            stream.append((k * 3 * W + W, m))  # the run goes on one whole tile later
        prev = m
    stream.append((40 * W, 1 << (ngroups - 1)))
    masked = [stream[3][0], stream[20][0]]
    s = Src(risect, codec, stream_lists(stream, ngroups), 41 * W, masked)
    tok = [[f"g{g}"] for g in range(ngroups)]
    got = s.check(tok)
    gd = [[d for d, m in stream if (m >> g) & 1] for g in range(ngroups)]
    assert dict(got) == consider_sequential([m for _, m in considered_stream(gd, masked)])
    assert any(m >> (ngroups - 1) for m, _ in got)


def limit_corpus():
    """17 groups; documents 1 .. 65 537 each with its own mask, the 17 masks of popcount 16 first (every later mask is a subset of one
    of them: the antichain stays at 17 entries).  Terms g<i> hold every document, h<i> all but the last: a request over the g terms has
    65 537 distinct considered masks, one over the h terms 65 536.  The full mask is origMask and never occurs."""
    full = (1 << 17) - 1
    top = [full ^ (1 << b) for b in range(17)]
    rest = [m for m in range(1, full) if bin(m).count("1") < 16]
    random.Random(3).shuffle(rest)
    masks = np.array(top + rest[: MAX_MASKS + 1 - 17], np.uint64)
    docs = np.arange(1, len(masks) + 1, dtype=np.uint32)
    lists = {}
    for g in range(17):
        has = docs[((masks >> np.uint64(g)) & np.uint64(1)).astype(bool)]
        lists[f"g{g}"] = has
        lists[f"h{g}"] = has[has < docs[-1]]
    return lists, len(masks)


@CODECS
def test_distinct_mask_limit(risect, codec):
    lists, n = limit_corpus()
    assert n == MAX_MASKS + 1
    s = Src(risect, codec, lists, n + 1)
    good = [["g0"], ["g1", "h2"], ["g3"]]
    at_limit = [[f"h{g}"] for g in range(17)]
    over = [[f"g{g}"] for g in range(17)]
    with pytest.raises(tb.TrinityError, match="rc=-6: .*request 2 has more than 65536 distinct"):
        s.gpu.intersect_batch([s.ids(good), s.ids(at_limit), s.ids(over)])
    res = s.gpu.intersect_batch([s.ids(good), s.ids(at_limit)])
    g0 = s.check(good, res[0])
    got = s.check(at_limit, res[1])
    assert res.distinct == s.gpu.intersect_batch([s.ids(good)]).distinct + MAX_MASKS
    assert sorted(got) == sorted((((1 << 17) - 1) ^ (1 << b), 1) for b in range(17))
    assert s.gpu.intersect(s.ids(good)) == g0  # the context stays usable


@CODECS
def test_table_bound_from_the_documents(risect, codec):
    """every document its own mask: the table is sized from the documents (postings), not from the limit or 2^groups - 1; single-bit
    masks (bound == distinct masks exactly) and two-bit masks over 64 groups"""
    ones = [(1 + 3 * g, 1 << g) for g in range(64)]
    pairs = [(1000 + 5 * i, (1 << a) | (1 << b)) for i, (a, b) in enumerate((a, b) for a in range(64) for b in range(a + 1, 64))]
    for stream in (ones, ones + pairs):
        s = Src(risect, codec, stream_lists(stream, 64), stream[-1][0] + 1)
        tok = [[f"g{g}"] for g in range(64)]
        res = s.gpu.intersect_batch([s.ids(tok)])
        got = s.check(tok, res[0])
        assert res.distinct == len(stream) and res.postings == sum(bin(m).count("1") for _, m in stream)
        assert dict(got) == consider_sequential([m for _, m in stream])
        assert got == finalize_order(got)
