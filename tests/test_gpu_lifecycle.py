"""A GpuIndexSource frees all its device memory when it closes, and its docID sets keep their memory while the table that holds them grows.
The GPU may be shared, so the leak check reads the free memory right around its cycles."""
import numpy as np
import pytest
import torch

import trinity_b200 as tb

pytestmark = pytest.mark.gpu

MiB = 1 << 20


def corpus(codec, ndocs, vocab, length, positions, seed):
    """ndocs documents of `length` tokens drawn uniformly from the vocabulary, indexed on the device; positions: token i at 1 + 255 i"""
    rng = np.random.default_rng(seed)
    tok = rng.integers(0, vocab, ndocs * length, dtype=np.uint32)
    offs = np.arange(ndocs + 1, dtype=np.uint64) * length
    pos = np.tile(1 + 255 * np.arange(length, dtype=np.uint32), ndocs) if positions else None
    gpu = tb.GpuIndexSource()
    try:
        return gpu.index_documents_flat(codec, np.arange(1, ndocs + 1, dtype=np.uint32), offs, tok, vocab, pos)
    finally:
        gpu.close()


def test_close_frees_device_memory():
    vocab, cycles = 4096, 8
    seg = corpus(tb.CODEC_LUCENE, 1_200_000, vocab, 64, True, seed=7)
    assert cycles * len(seg.hits) >= 1 << 30, len(seg.hits)
    names = [f"t{i}" for i in range(vocab)]
    texts = ["t1 AND t2", "t3 OR t4", "t5 AND (t6 OR t7)"]

    def cycle():
        gpu = tb.GpuIndexSource()
        try:
            tdict = seg.upload(gpu, names)
            plans = [tb.parse_query(t, tdict) for t in texts]
            docs = gpu.exec_batch(plans, tb.MODE_DOCS_COMPACT)
            m = gpu.exec_matches(plans[:2])
            return [docs.query(q)[0] for q in range(len(texts))], [m.query(q) for q in range(2)]
        finally:
            gpu.close()

    want_docs, want_matches = cycle()  # the CUDA context and the modules are paid for here
    assert all(len(d) for d in want_docs)
    free0, _ = torch.cuda.mem_get_info()
    for i in range(cycles):
        docs, matches = cycle()
        assert all(np.array_equal(a, b) for a, b in zip(docs, want_docs)), f"cycle {i}: documents"
        assert all(np.array_equal(a, b) for a, b in zip(matches, want_matches)), f"cycle {i}: matches"
    free1, _ = torch.cuda.mem_get_info()
    lost = (free0 - free1) / MiB
    assert lost < 256, f"{cycles} cycles of a {len(seg.hits) / MiB:.0f} MiB hits.data lost {lost:.0f} MiB of device memory"


def test_docsets_survive_table_growth():
    ndocs, vocab = 20_000, 64
    seg = corpus(tb.CODEC_GOOGLE, ndocs, vocab, 32, False, seed=11)
    rng = np.random.default_rng(12)
    gpu = tb.GpuIndexSource()
    try:
        tdict = seg.upload(gpu, [f"t{i}" for i in range(vocab)])
        members = [np.unique(rng.integers(1, ndocs + 1, ndocs // 3)) for _ in range(100)]  # a doubling table reallocates 7 times
        sets = [gpu.docset(m) for m in members]
        plans = [tb.parse_query(t, tdict) for t in ("t1 AND t2", "t3 OR t4", "t5 AND (t6 OR t7)")]
        cases = [(0, "allow"), (-1, "allow"), (0, "deny"), (-1, "deny")]
        batch = [p for p in plans for _ in cases]
        filters = [tb.DocFilter(**{side: sets[s]}) for _ in plans for s, side in cases]
        got = gpu.exec_batch(batch, tb.MODE_DOCS_ONLY, filters=filters)
        plain = gpu.exec_batch(batch, tb.MODE_DOCS_ONLY)
        for i in range(len(batch)):
            s, side = cases[i % len(cases)]
            d = plain.query(i)[0]
            want = d[np.isin(d, members[s], invert=side == "deny")]
            assert len(want) and np.array_equal(got.query(i)[0], want), f"query {i}: set {s} as {side}"
    finally:
        gpu.close()
