"""The merge planner (csrc/mergeplan.h, trn_debug_merge_plan) against a Python restatement of merge.cpp's candidate order, term loop and
routes; consider_tracked_sources against the reference's.  No GPU."""
import numpy as np
import pytest

import trinity_b200 as tb
from trinity_b200._ffi import TERM_DTYPE
from mergeutil import model_plan, ref_consider_tracked_sources


def _src(codec, gen, names, docs, upd=(), rng=None):
    terms = np.zeros(len(names), TERM_DTYPE)
    terms["documents"] = docs
    return tb.MergeSource(codec, gen, np.zeros(16, np.uint8), terms, names, np.zeros(0, np.uint8) if codec == tb.CODEC_LUCENE else None,
                          np.asarray(upd, np.uint32))


def _check(out_codec, sources, disable):
    got = tb.debug_merge_plan(out_codec, sources, disable)
    want = model_plan(out_codec, sources, disable)
    assert got["order"] == want["order"]
    assert got["route"] == want["route"] and got["stats"] == want["stats"]
    off = got["part_off"]
    assert [got["parts"][off[k]:off[k + 1]] for k in range(len(off) - 1)] == want["parts"]
    assert got["upd_docid"] == want["upd_docid"] and got["upd_first"] == want["upd_first"]
    assert got["countdown_phase"] == 0


def _terms_cmp_sorted(names):
    return sorted(set(names), key=lambda n: n.encode())


@pytest.mark.parametrize("seed", range(1000))
def test_plan_equals_the_model_on_random_name_sets(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 6))
    pool = ["a", "ab", "abc", "b", "ba", "z", "zz"] + [f"t{i}" for i in range(int(rng.integers(1, 40)))]
    gens = rng.choice(np.arange(1, 100), n, replace=False)
    sources = []
    for s in range(n):
        names = _terms_cmp_sorted(rng.choice(pool, int(rng.integers(0, len(pool))), replace=True).tolist())
        docs = rng.integers(0, 3, len(names))
        upd = rng.choice(np.arange(1, 50), int(rng.integers(0, 4)), replace=False) if rng.random() < 0.5 else []
        sources.append(_src(int(rng.integers(0, 2)), int(gens[s]), names, docs, upd))
    _check(int(rng.integers(0, 2)), sources, bool(rng.integers(0, 2)))


def test_routes_on_the_named_shapes():
    G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE
    old = _src(G, 1, ["a", "ab", "only_old", "zero"], [3, 2, 4, 0])
    new = _src(G, 2, ["a", "b", "only_new"], [1, 5, 2], upd=[7])
    plan = tb.debug_merge_plan(G, [old, new])
    # names merged in terms_cmp order: a (2 holders), ab (old, masked by the newer one's update: re-encode), b, only_new (appends), only_old
    assert plan["order"] == [1, 0]
    assert plan["route"] == [1, 1, 0, 0, 1]
    assert plan["stats"] == [0, 1, 0, 0, 1]
    assert tb.debug_merge_plan(L, [old, new])["route"] == [1, 1, 1, 1, 1]
    assert tb.debug_merge_plan(G, [old, new], True)["stats"] == [1, 1, 1, 1, 1]
    assert tb.debug_merge_plan(G, [])["route"] == []


def test_planner_refusals():
    G = tb.CODEC_GOOGLE
    with pytest.raises(tb.TrinityError, match="share generation"):
        tb.debug_merge_plan(G, [_src(G, 3, ["a"], [1]), _src(G, 3, ["b"], [1])])
    with pytest.raises(tb.TrinityError, match="at most 128"):
        tb.debug_merge_plan(G, [_src(G, g + 1, ["a"], [1]) for g in range(129)])
    with pytest.raises(tb.TrinityError, match="strictly ascending"):
        tb.debug_merge_plan(G, [_src(G, 1, ["b", "a"], [1, 1])])
    with pytest.raises(tb.TrinityError, match="1 to 64 bytes"):
        tb.debug_merge_plan(G, [_src(G, 1, ["x" * 65], [1])])
    s = _src(G, 1, ["a"], [1])
    s.terms["chunk_len"] = 17
    with pytest.raises(tb.TrinityError, match="outside the source"):
        tb.debug_merge_plan(G, [s])
    with pytest.raises(tb.TrinityError, match="hits.data"):
        tb.debug_merge_plan(G, [tb.MergeSource(tb.CODEC_LUCENE, 1, np.zeros(16, np.uint8), s.terms, ["a"], None, None)])
    assert len(tb.debug_merge_plan(G, [_src(G, g + 1, ["a"], [1]) for g in range(128)])["order"]) == 128


@pytest.mark.parametrize("seed", range(50))
def test_consider_tracked_sources_equals_the_reference(seed):
    rng = np.random.default_rng(seed)
    tracked = rng.choice(np.arange(1, 40), int(rng.integers(0, 12)), replace=False).tolist()
    cands = [g for g in tracked if rng.random() < 0.6] + rng.choice(np.arange(40, 50), int(rng.integers(0, 2)), replace=False).tolist()
    assert tb.consider_tracked_sources(cands, tracked) == ref_consider_tracked_sources(cands, tracked)
