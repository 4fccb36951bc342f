"""How trn_exec_batch splits a batch into pipelined launches (csrc/chunkplan.h, the function the engine itself calls) on the benchmark's
scenarios: first batch of a shape by referenced postings; afterwards by the previous batch's
result size, c = sqrt(D / 4 tail), the last chunk tapered into 1/2, 1/4, 1/4."""
import ctypes as C

import numpy as np
import pytest

from trinity_b200._ffi import lib


def plan(nq, est, leaves, hint_bytes=0, hint_postings=0, same=False, topk=False, max_chunks=8, chunk_postings=10**9, rule_sqrt=True, taper=True,
         tail_ms=0.15, tail_tree_ms=0.9):
    sizes = np.zeros(32, np.uint32)
    n, single = C.c_uint32(), C.c_int()
    rc = lib().trn_debug_chunk_plan(nq, int(topk), est, leaves, max_chunks, chunk_postings, int(rule_sqrt), int(taper), tail_ms, tail_tree_ms, hint_bytes,
                                    hint_postings, int(same), sizes.ctypes.data_as(C.c_void_p), 32, C.byref(n), C.byref(single))
    assert rc == 0
    out = [int(x) for x in sizes[: n.value]]
    assert sum(out) == nq and all(x > 0 for x in out)
    return bool(single.value), out


AND2 = dict(nq=1000, est=17_500_000_000, leaves=2000)          # the headline batch, unsharded: 1.75e10 referenced postings
AND2_SHARD = dict(nq=1000, est=2_190_000_000, leaves=2000)     # ... on one of 8 docID shards
TREE8 = dict(nq=1000, est=70_000_000_000, leaves=8000)
TREE8_SHARD = dict(nq=1000, est=8_750_000_000, leaves=8000)


def test_first_batch_of_a_shape_goes_by_referenced_postings():
    single, s = plan(**AND2)
    assert not single and s == [125] * 7 + [62, 31, 32]          # 8 chunks, the last one tapered
    single, s = plan(**AND2_SHARD)
    assert not single and s == [500, 250, 125, 125]              # 2 chunks + taper
    single, s = plan(nq=64, est=5_000, leaves=128)               # tiny index: nothing to pipeline
    assert single and s == [64]
    single, s = plan(nq=64, est=5_000, leaves=128, chunk_postings=1)  # (the test suite forces chunks this way)
    assert not single and len(s) == 8


def test_result_size_rule_on_the_measured_scenarios():
    # and2 at N = 1: 0.675 GB out -> D = 15 ms, tail 0.15 -> 5 chunks + taper
    single, s = plan(**AND2, hint_bytes=674_787_528, hint_postings=AND2["est"], same=True)
    assert not single and len(s) == 7 and s[:4] == [200] * 4 and s[4:] == [100, 50, 50]
    # one of 8 shards: 92.6 MB -> D = 2.06 ms -> 2 chunks + taper
    single, s = plan(**AND2_SHARD, hint_bytes=92_574_116, hint_postings=AND2_SHARD["est"], same=True)
    assert not single and s == [500, 250, 125, 125]
    # tree8 at N = 1: 0.54 GB, tree tail 0.9 ms -> 2 chunks + taper
    single, s = plan(**TREE8, hint_bytes=540_682_420, hint_postings=TREE8["est"], same=True)
    assert not single and s == [500, 250, 125, 125]
    # tree8 on one of 8 shards: 67 MB = 1.5 ms of copy is not worth two 0.9 ms tails -> one call
    single, s = plan(**TREE8_SHARD, hint_bytes=67_373_840, hint_postings=TREE8_SHARD["est"], same=True)
    assert single and s == [1000]
    # a lone chunk whose copy IS worth two launches is still tapered (and2 shard with a 0.3 ms tail)
    single, s = plan(**AND2_SHARD, hint_bytes=92_574_116, hint_postings=AND2_SHARD["est"], same=True, tail_ms=0.3)
    assert not single and s == [500, 250, 250]


def test_hint_of_another_shape_is_ignored_and_knobs_hold():
    base = plan(**AND2)
    assert plan(**AND2, hint_bytes=10**9, hint_postings=AND2["est"], same=False) == base                # other nq / mode
    assert plan(**AND2, hint_bytes=10**9, hint_postings=AND2["est"] * 2, same=True) == base             # postings differ by more than 25 %
    assert plan(**AND2, hint_bytes=10**9, hint_postings=AND2["est"], same=True, rule_sqrt=False) == base  # TRN_CHUNK_RULE=postings
    single, s = plan(**AND2, taper=False)
    assert not single and s == [125] * 8
    single, s = plan(**AND2, max_chunks=1)
    assert single
    single, s = plan(**AND2, topk=True)
    assert single and s == [1000]
    single, s = plan(nq=40, est=10**11, leaves=80)        # fewer than 8 queries per chunk: one call
    assert single
    single, s = plan(**AND2, hint_bytes=10**12, hint_postings=AND2["est"], same=True)  # capped at TRN_PIPELINE_CHUNKS
    assert not single and len(s) == 10
