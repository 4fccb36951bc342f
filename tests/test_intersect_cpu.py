"""Query-token intersections on the CPU: the sequential transcription of ctx::consider against the reference's intersect() on small sources
of both codecs, the epoch restatement the device passes implement against the sequential one on random streams, and the host planner
(trn_debug_intersect_plan) against its Python twin, with its mask limit."""
import random

import numpy as np
import pytest

import trinity_b200 as tb
from isectutil import RefIsect, considered_stream, consider_epochs, consider_sequential, epoch_plan

CODECS = pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])


def random_stream(rng, ngroups, ndocs):
    """[(docID, mask)] with docIDs ascending and masks over ngroups bits, runs of equal masks likely"""
    out, d, m = [], 0, 0
    for _ in range(ndocs):
        d += rng.randint(1, 3)
        if m == 0 or rng.random() < 0.6:
            m = rng.randint(1, (1 << ngroups) - 1)
        out.append((d, m))
    return out


@pytest.fixture(scope="module")
def risect():
    return RefIsect()


def small_source(codec, seed, nterms=8, ndocs=3000):
    rng = np.random.default_rng(seed)
    names, lists = [f"k{i}" for i in range(nterms)], []
    b = tb.IndexBuilder(codec)
    for i in range(nterms):
        df = int(rng.integers(1, ndocs // (i + 2)))
        d = np.sort(rng.choice(np.arange(1, ndocs), size=df, replace=False)).astype(np.uint32)
        lists.append(d)
        b.add_term(d, np.ones(df, np.uint32))
    return names, lists, b.index(), b.terms_array(), b.hits()


@CODECS
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_sequential_transcription_equals_reference(risect, codec, seed):
    names, lists, index, terms, hits = small_source(codec, seed)
    src = risect.source(codec, index, names, terms, hits)
    rng = random.Random(seed)
    masked = sorted(rng.sample(range(1, 3000), 200))
    for _ in range(12):
        ng = rng.randint(1, 6)
        groups = [rng.sample(range(len(names)), rng.randint(1, 2)) for _ in range(ng)]
        unknown = rng.random() < 0.2
        tok = [[names[t] for t in g] for g in groups]
        if unknown:
            tok[0].append("nosuchtoken")
        gd = [np.union1d(lists[g[0]], lists[g[-1]]) for g in groups]
        orig = 0 if unknown else None
        for mk in ((), masked):
            want = dict(src.intersect(tok, mk))
            got = consider_sequential([m for _, m in considered_stream(gd, mk, orig)])
            assert got == want, (tok, bool(mk))


def test_sequential_transcription_all_unknown(risect):
    names, lists, index, terms, _ = small_source(tb.CODEC_GOOGLE, 4)
    src = risect.source(tb.CODEC_GOOGLE, index, names, terms)
    assert src.intersect([["nosuch"], ["other"]]) == []


def test_epoch_restatement_equals_sequential():
    rng = random.Random(0x15EC7)
    for _ in range(10_000):
        s = random_stream(rng, rng.randint(1, 6), rng.randint(1, 60))
        assert consider_epochs(s) == consider_sequential([m for _, m in s]), s


def test_epoch_restatement_wide_antichain():
    """more than 256 incomparable masks: the reference's indexPrev is a uint8_t, so a run continued on an entry past 255 adds to entry
    index & 255 — the restatement follows it"""
    rng = random.Random(7)
    pairs = [(1 << a) | (1 << b) for a in range(30) for b in range(a + 1, 30)]  # 435 two-bit masks
    rng.shuffle(pairs)
    s, d = [], 0
    for m in pairs + pairs[:100] + [1 << 3, 1 << 7]:
        for _ in range(rng.randint(1, 4)):
            d += 1
            s.append((d, m))
    seq = consider_sequential([m for _, m in s])
    assert consider_epochs(s) == seq
    assert len(seq) == 435


def test_debug_plan_equals_python_planner():
    rng = random.Random(99)
    for _ in range(2000):
        s = random_stream(rng, rng.randint(1, 7), rng.randint(1, 80))
        first = {}
        for d, m in s:
            first.setdefault(m, d)
        masks, firsts = list(first), list(first.values())
        order = list(range(len(masks)))
        rng.shuffle(order)  # the planner orders the masks by their first docID itself
        got = tb.debug_intersect_plan([masks[i] for i in order], [firsts[i] for i in order])
        starts, arrays, final = epoch_plan(masks, firsts)
        assert got == (starts, arrays, final)


def test_debug_plan_mask_limit():
    masks = list(range(1, 1001))
    firsts = list(range(10, 10010, 10))
    _, _, final = tb.debug_intersect_plan(masks, firsts, max_masks=1000)
    assert final
    with pytest.raises(tb.TrinityError, match="rc=-6"):
        tb.debug_intersect_plan(masks, firsts, max_masks=999)
    with pytest.raises(tb.TrinityError, match="rc=-6"):
        tb.debug_intersect_plan(list(range(1, 65538)), list(range(1, 65538)))  # the default limit: 65536
    tb.debug_intersect_plan(list(range(1, 65537)), list(range(1, 65537)))
