"""trn_merge_sources against the reference's MergeCandidatesCollection::merge() over the same generations (written by the reference's
SegmentIndexSession, with replaced and erased documents): every file of the merged directory (LUCENE: except the PFor padding the
reference leaves uninitialised), both output codecs, disableOptimizations on and off; refusals that leave the context usable."""
import numpy as np
import pytest

import trinity_b200 as tb
from idxutil import read_dir, ref_index
from mergeutil import random_specs, ref_merge, write_generation
from idxutil import flat, zipf_corpus
from test_merge_model_cpu import SHAPES as HOST_SHAPES
from trinity_b200.segments import SegmentCollection

pytestmark = pytest.mark.gpu
G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE


def _same_but_padding(mine, theirs, what):
    assert mine.size == theirs.size, what
    diff = np.flatnonzero(mine != theirs)
    assert np.all(mine[diff] == 0), f"{what} differs at non-padding bytes {diff[:10]}"


def make_generations(root, codecs, ndocs, nterms, seed, max_docid=None, long_docs=False):
    """len(codecs) generations, oldest first: each indexes new documents, replaces some older ones and erases a few.  Returns the paths
    and the surviving (docID -> generation index) map."""
    rng = np.random.default_rng(seed)
    names = sorted({f"t{i}" for i in range(nterms)} | {"t", "t1x", "zz"}, key=str.encode)
    hi = max_docid or ndocs * 4
    live, paths, ever = {}, [], set()
    for g, codec in enumerate(codecs):
        fresh = rng.choice(hi, ndocs, replace=False) + 1
        fresh = [int(d) for d in fresh if int(d) not in ever][: ndocs // 2]
        older = sorted(live)
        repl = [int(d) for d in rng.choice(older, min(len(older), ndocs // 4), replace=False)] if older else []
        ers = [d for d in older if d not in repl and rng.random() < 0.05]
        docids = fresh + repl
        docs, pos = [], []
        w = 1.0 / np.arange(1, len(names) + 1)
        for i, _ in enumerate(docids):
            if long_docs and i == 0:  # 17 000 hits of one term in one document, at positions 1..16383 (equal positions allowed)
                docs.append(np.zeros(17000, np.uint32))
                pos.append((np.arange(17000) % 16383 + 1).astype(np.uint32))
                continue
            n = int(rng.integers(1, 24))
            docs.append(rng.choice(len(names), n, p=w / w.sum()).astype(np.uint32))
            pos.append(np.arange(1, n + 1, dtype=np.uint32))
        p = root / f"{g + 1}"
        ref_index(codec, p, names, docids, docs, pos, replaced=repl, erased=ers)
        for d in ers:
            live.pop(d, None)
        for d in docids:
            live[d] = g
        ever.update(docids)
        paths.append(p)
    return paths, live


def _compare(got_dir, want_dir, codec):
    want, got = read_dir(want_dir), read_dir(got_dir)
    assert sorted(want) == sorted(got)
    for f in want:
        if codec == L and f in ("index", "hits.data"):
            _same_but_padding(got[f], want[f], f)
        else:
            assert np.array_equal(got[f], want[f]), f


def _merge_both(tmp_path, paths, out_codec, disable, tag):
    coll = SegmentCollection(paths)
    m = coll.merge(out_codec, disable)
    ref_fs, _ = ref_merge(out_codec, tmp_path / f"ref{tag}" / "100", paths, disable, m.field_statistics["docsCnt"])
    assert m.field_statistics == ref_fs
    m.write(tmp_path / f"dev{tag}" / "100")
    _compare(tmp_path / f"dev{tag}" / "100", tmp_path / f"ref{tag}" / "100", out_codec)
    return m


SHAPES = {"one": [G], "one_lucene": [L], "two": [G, G], "three": [G, L, G], "eight": [L, G, L, L, G, G, L, G], "lucene3": [L, L, L]}


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("out_codec", [G, L], ids=["google", "lucene"])
@pytest.mark.parametrize("disable", [False, True], ids=["opt", "noopt"])
def test_merge_equals_the_reference(tmp_path, shape, out_codec, disable):
    paths, live = make_generations(tmp_path / "src", SHAPES[shape], 400, 150, seed=len(shape) * 7 + out_codec)
    m = _merge_both(tmp_path, paths, out_codec, disable, "")
    assert m.field_statistics["docsCnt"] == len(live)


@pytest.mark.parametrize("out_codec", [G, L], ids=["google", "lucene"])
def test_high_docids_and_long_documents(tmp_path, out_codec):
    paths, live = make_generations(tmp_path / "src", [G, L, G], 300, 40, seed=5, max_docid=2**32 - 2, long_docs=True)
    assert max(live) > 2**31
    for disable in (False, True):
        m = _merge_both(tmp_path, paths, out_codec, disable, str(int(disable)))
        assert m.field_statistics["docsCnt"] == len(live)


def test_merged_segment_answers_like_the_collection(ref, tmp_path):
    # GOOGLE generations: SegmentCollection runs phrases on sources whose hits are inline
    paths, _ = make_generations(tmp_path / "src", [G, G, G], 500, 60, seed=11)
    coll = SegmentCollection(paths)
    m = coll.merge(G)
    m.write(tmp_path / "m" / "100")
    merged = SegmentCollection([tmp_path / "m" / "100"])
    for q in ("t1", "t2 AND t3", "t1 OR t7", "\"t0 t1\"", "t4 NOT t2"):
        want = set()
        for r in coll.exec_batch([q], tb.MODE_DOCS_ONLY):
            want |= set(r.query(0)[0].tolist())
        got = set(merged.exec_batch([q], tb.MODE_DOCS_ONLY)[0].query(0)[0].tolist())
        assert got == want, q
        # the reference's own SegmentIndexSource over the merged directory agrees
        assert set(ref.segment_open(tmp_path / "m" / "100").exec(q, False, 1 << 22)[0].tolist()) == want, q


def test_refusals_leave_the_context_usable(tmp_path):
    paths, _ = make_generations(tmp_path / "src", [G, G], 200, 30, seed=3)
    coll = SegmentCollection(paths)
    srcs = [tb.MergeSource.of_segment(s, p, g) for s, p, g in zip(coll.segments, coll.paths, coll.generations)]
    g = tb.GpuIndexSource(0)
    try:
        first = g.merge_sources(G, srcs)
        with pytest.raises(tb.TrinityError, match="at most 128"):
            g.merge_sources(G, [tb.MergeSource(G, i + 1, srcs[0].index, srcs[0].terms, srcs[0].names) for i in range(129)])
        with pytest.raises(tb.TrinityError, match="share generation"):
            g.merge_sources(G, [srcs[0], srcs[0]])
        again = g.merge_sources(G, srcs)
        assert np.array_equal(first.index, again.index) and first.names == again.names
        many = g.merge_sources(G, [tb.MergeSource(G, i + 1, srcs[0].index, srcs[0].terms, srcs[0].names) for i in range(128)])
        assert many.field_statistics["totalTerms"] == len(srcs[0].names)
        assert len(g.merge_sources(G, []).index) == 0
    finally:
        g.close()


def _host_sources(root, codecs, seed, **kw):
    specs, updated = random_specs(np.random.default_rng(seed), codecs, **kw)
    paths = [root / f"{g + 1}" for g in range(len(codecs))]
    return paths, [write_generation(p, c, s, u) for p, c, s, u in zip(paths, codecs, specs, updated)]


@pytest.mark.parametrize("shape", list(HOST_SHAPES))
@pytest.mark.parametrize("out_codec", [G, L], ids=["google", "lucene"])
@pytest.mark.parametrize("disable", [False, True], ids=["opt", "noopt"])
@pytest.mark.parametrize("kind", ["plain", "freq0"])
def test_host_built_generations(tmp_path, shape, out_codec, disable, kind):
    """the shapes of test_merge_model_cpu (prefix names, > 64 terms, lists of many blocks between appended terms, an orphan term,
    freq-0 LUCENE postings) on the device, against the reference"""
    paths, srcs = _host_sources(tmp_path / "src", HOST_SHAPES[shape], seed=len(shape) * 31 + out_codec, freq0=kind == "freq0")
    g = tb.GpuIndexSource(0)
    try:
        m = g.merge_sources(out_codec, srcs, disable)
    finally:
        g.close()
    ref_fs, _ = ref_merge(out_codec, tmp_path / "ref" / "100", paths, disable, m.field_statistics["docsCnt"])
    assert m.field_statistics == ref_fs
    m.write(tmp_path / "dev" / "100")
    _compare(tmp_path / "dev" / "100", tmp_path / "ref" / "100", out_codec)
    if len(paths) >= 3:
        assert m.counts["orphaned"] >= 1
    if kind == "freq0" and L in HOST_SHAPES[shape]:
        assert m.field_statistics["sumTermsDocs"] == 0 or m.counts["postings_written"] > 0


def test_payloads(tmp_path):
    """re-encoded payload hits are refused naming the term; appended chunks keep their payloads byte for byte"""
    paths, srcs = _host_sources(tmp_path / "src", [G, G], seed=9, payloads=True)
    g = tb.GpuIndexSource(0)
    try:
        with pytest.raises(tb.TrinityError, match=r"rc=-\d+: trn_merge_sources: source \d \(generation \d\), term \[.*\]: a hit with a payload"):
            g.merge_sources(G, srcs, True)
        p1, s1 = _host_sources(tmp_path / "one", [G], seed=10, payloads=True)
        for out_codec in (G,):
            m = g.merge_sources(out_codec, s1)
            assert m.counts["reencoded"] == 0 and m.counts["appended"] == len(s1[0].names)
            ref_merge(out_codec, tmp_path / "ref" / "100", p1, False, m.field_statistics["docsCnt"])
            m.write(tmp_path / "dev" / "100")
            _compare(tmp_path / "dev" / "100", tmp_path / "ref" / "100", out_codec)
    finally:
        g.close()


def test_128_sources_equal_the_reference(tmp_path):
    rng = np.random.default_rng(12)
    paths, srcs = [], []
    for i in range(128):
        spec = {f"t{int(t)}": [(int(d), [(1, b"")]) for d in sorted(rng.choice(5000, 3, replace=False) + 1)] for t in rng.choice(20, 4, replace=False)}
        p = tmp_path / "src" / f"{i + 1}"
        srcs.append(write_generation(p, G if i % 3 else L, spec, rng.choice(5000, 2, replace=False) + 1))
        paths.append(p)
    g = tb.GpuIndexSource(0)
    try:
        m = g.merge_sources(G, srcs)
    finally:
        g.close()
    ref_fs, _ = ref_merge(G, tmp_path / "ref" / "100", paths, False, m.field_statistics["docsCnt"])
    assert m.field_statistics == ref_fs
    m.write(tmp_path / "dev" / "100")
    _compare(tmp_path / "dev" / "100", tmp_path / "ref" / "100", G)


def test_every_refusal_keeps_the_context(tmp_path):
    """each refusal names the source; the next good call gives the earlier result; an uploaded index and a percolator registry stay"""
    paths, srcs = _host_sources(tmp_path / "src", [G, L], seed=4)
    names = [f"t{i}" for i in range(8)]
    g = tb.GpuIndexSource(0)
    try:
        rng = np.random.default_rng(1)
        docs = [rng.integers(0, 8, 10).astype(np.uint32) for _ in range(500)]
        seg = g.index_documents(G, np.arange(1, 501, dtype=np.uint32), docs, 8)
        tdict = seg.upload(g, names)
        plans = [tb.parse_query("t1 AND t2", tdict)]
        g.percolator_register([tb.parse_query("t1 AND t2", tb.TermDictionary(names))], 8)
        before, pbefore = g.exec_batch(plans, tb.MODE_DOCS_ONLY).query(0)[0].copy(), g.percolate(docs[:50]).queries.copy()
        first = g.merge_sources(L, srcs)
        bad_order = tb.MergeSource(G, 7, srcs[0].index, srcs[0].terms[::-1].copy(), list(srcs[0].names)[::-1])
        empty_name = tb.MergeSource(G, 7, srcs[0].index, srcs[0].terms, [""] + list(srcs[0].names[1:]))
        outside = srcs[0].terms.copy()
        outside["chunk_off"][0] = len(srcs[0].index)
        no_hits = tb.MergeSource(L, 7, srcs[1].index, srcs[1].terms, srcs[1].names, None)
        cases = [([bad_order], "strictly ascending"), ([empty_name], "1 to 64 bytes"),
                 ([tb.MergeSource(G, 7, srcs[0].index, outside, srcs[0].names)], "outside the source"), ([no_hits], "hits.data"),
                 ([srcs[0], srcs[0]], "share generation"),
                 ([tb.MergeSource(G, i + 1, srcs[0].index, srcs[0].terms, srcs[0].names) for i in range(129)], "at most 128")]
        for bad, msg in cases:
            with pytest.raises(tb.TrinityError, match=msg):
                g.merge_sources(L, bad)
            again = g.merge_sources(L, srcs)
            assert np.array_equal(again.index, first.index) and np.array_equal(again.hits, first.hits) and again.names == first.names
        assert np.array_equal(g.exec_batch(plans, tb.MODE_DOCS_ONLY).query(0)[0], before)
        assert np.array_equal(g.percolate(docs[:50]).queries, pbefore)
        assert len(g.merge_sources(G, []).index) == 0
    finally:
        g.close()


@pytest.mark.parametrize("out_codec", [G, L], ids=["google", "lucene"])
def test_zipf_device_indexed_generations(tmp_path, out_codec):
    """4 device-indexed generations x 250 000 documents x 64 tokens, 10 % of each replacing older documents, some erased"""
    names = sorted([f"w{i}" for i in range(2000)], key=str.encode)
    g = tb.GpuIndexSource(0)
    paths, live = [], set()
    try:
        for k in range(4):
            docids, offs, tok = zipf_corpus(250_000, len(names), 64, seed=100 + k)
            docids = docids + np.uint32(225_000 * k)  # 25 000 of each generation's docIDs are the previous one's
            older = np.array(sorted(live), np.uint32)
            replaced = np.intersect1d(docids, older)
            erased = np.setdiff1d(older[::97], docids)
            seg = g.index_documents_flat(L if k % 2 else G, docids, offs, tok, len(names))
            p = tmp_path / "src" / f"{k + 1}"
            seg.write(p, names, replaced=replaced, erased=erased)
            paths.append(p)
            live = (live - set(erased.tolist())) | set(docids.tolist())
    finally:
        g.close()
    for disable in (False, True):
        m = SegmentCollection(paths).merge(out_codec, disable)
        assert m.field_statistics["docsCnt"] == len(live)
        ref_fs, _ = ref_merge(out_codec, tmp_path / f"ref{int(disable)}" / "100", paths, disable, m.field_statistics["docsCnt"])
        assert m.field_statistics == ref_fs
        m.write(tmp_path / f"dev{int(disable)}" / "100")
        _compare(tmp_path / f"dev{int(disable)}" / "100", tmp_path / f"ref{int(disable)}" / "100", out_codec)
