"""The host encoders (codecs.cpp, IndexBuilder.new_hit with a payload) against the reference Encoders on the payload shapes the device
encoders are checked with (tests/test_gpu_payloads.py): GOOGLE byte for byte, LUCENE byte for byte except the PFor padding the reference
leaves uninitialised."""
import numpy as np
import pytest

import trinity_b200 as tb
from matchutil import host_build, ref_build
from payutil import google_shapes, lucene_shapes

SHAPES = {tb.CODEC_GOOGLE: google_shapes, tb.CODEC_LUCENE: lucene_shapes}


def _same_but_padding(mine, theirs, what):
    assert mine.size == theirs.size, what
    diff = np.flatnonzero(mine != theirs)
    # the reference leaves the padding of the PFor byte container uninitialised (fastpfor.h:196-198): only there, and only zeros of ours
    assert np.all(mine[diff] == 0), f"{what} differs at non-padding bytes {diff[:10]}"


@pytest.mark.parametrize("codec", [tb.CODEC_GOOGLE, tb.CODEC_LUCENE], ids=["google", "lucene"])
def test_host_encoder_payloads_equal_the_reference_encoder(codec):
    shapes = SHAPES[codec](np.random.default_rng(41))
    lists = [l for _, l in shapes]
    index, hits, terms = host_build(codec, lists)
    r = ref_build(codec, lists, [n for n, _ in shapes], int(max(int(l[0].max()) for l in lists if len(l[0]))))
    assert np.array_equal(terms, r.terms())
    if codec == tb.CODEC_GOOGLE:
        assert np.array_equal(index, r.index()), f"first differing byte at {int(np.flatnonzero(index != r.index())[0])}"
        assert hits.size == 0
    else:
        _same_but_padding(index, r.index(), "index")
        _same_but_padding(hits, r.hits(), "hits.data")
    sizes = np.concatenate([l[3] for l in lists])
    assert set(np.unique(sizes).tolist()) == set(range(9))
