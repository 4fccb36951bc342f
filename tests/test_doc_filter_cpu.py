"""Per-query document filters on the CPU: the oracle the GPU tests use, the argument packing of the Python layer and the docID-set cache
of SegmentCollection.

The GPU tests take as the oracle of a filtered query the reference's exec_query with a masked_documents_registry that holds the masked
documents plus every document the filter drops.  Here that is checked against the reference's unfiltered run restricted on the host, on
both codecs and in both flag modes."""
import numpy as np
import pytest

import trinity_b200 as tb
from trinity_b200.segments import SegmentCollection
from util import Pair, closed_form_lists

NDOCS = 50_000
QUERIES = ["t1 AND t2", "t3 OR t7 OR t9", "t1 AND (t2 OR t3) NOT t5", "t10", "(t1 AND t2) OR (t3 AND t4)", "t2 AND t3 AND t5"]


@pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def test_oracle_registry_equals_restricted_unfiltered_run(ref, codec):
    p = Pair(ref, codec, closed_form_lists(NDOCS), NDOCS, upload=False)
    rng = np.random.default_rng(5)
    allow = np.unique(rng.integers(1, NDOCS + 1, NDOCS // 3)).astype(np.uint32)
    deny = np.arange(7, NDOCS + 1, 7, dtype=np.uint32)
    keep = np.zeros(NDOCS + 1, bool)
    keep[allow] = True
    keep[deny] = False
    ign = np.flatnonzero(~keep[1:]).astype(np.uint32) + 1
    for q in QUERIES:
        for scored in (False, True):
            d0, s0 = p.ref.exec(q, scored, NDOCS + 1)
            d1, s1 = p.ref.exec_masked(q, scored, ign, NDOCS + 1)
            m = keep[d0]
            assert np.array_equal(d1, d0[m]), (q, scored)
            if scored:
                assert np.array_equal(s1, s0[m]), q


class _FakeSource:
    def __init__(self):
        self.created = []

    def docset(self, d):
        self.created.append(np.asarray(d).copy())
        return tb.DocSet(self, len(self.created), len(d))


def test_pack_filters():
    src = _FakeSource()
    a, b = tb.DocSet(src, 3, 1), tb.DocSet(src, 7, 1)
    assert tb._pack_filters(None, 2) is None
    got = tb._pack_filters([None, tb.DocFilter(allow=a), tb.DocFilter(deny=b), tb.DocFilter(a, b)], 4, src)
    N = tb.DOCSET_NONE
    assert got.dtype == np.uint32 and got.tolist() == [[N, N], [3, N], [N, 7], [3, 7]]
    with pytest.raises(ValueError, match="filters for"):
        tb._pack_filters([None], 2)
    with pytest.raises(ValueError, match="another index source"):
        tb._pack_filters([tb.DocFilter(allow=a)], 1, _FakeSource())
    a.handle = None
    with pytest.raises(ValueError, match="closed"):
        tb._pack_filters([tb.DocFilter(allow=a)], 1)


def test_segment_collection_registers_and_caches_sets():
    c = SegmentCollection.__new__(SegmentCollection)  # the set bookkeeping only: no segments, no device
    c.sources = [_FakeSource(), _FakeSource(), _FakeSource()]
    c._docsets = {}
    assert c.filters(2) is None and c.filters(2, allow=[None, None]) is None
    f = c.filters(3, allow=[[5, 3, 3], None, [3, 5]], deny=[None, None, [9]])
    assert len(f) == 3 and all(len(x) == 3 for x in f)
    for i, s in enumerate(c.sources):
        # one set per distinct content in every source (generations share the docID space); [5, 3, 3] and [3, 5] are the same set
        assert [x.tolist() for x in s.created] == [[3, 5], [9]]
        assert f[i][1] is None
        assert f[i][0].allow is f[i][2].allow and f[i][0].allow.source is s
        assert f[i][0].deny is None and f[i][2].deny.source is s
    c.filters(1, deny=[[9]])
    assert all(len(s.created) == 2 for s in c.sources)  # passed again: reused
    with pytest.raises(ValueError):
        c.filters(2, allow=[None])
