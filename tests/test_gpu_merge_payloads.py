"""trn_merge_sources_payloads (GpuIndexSource.merge_sources(..., payloads=True), SegmentCollection.merge(..., payloads=True)) against the
reference's MergeCandidatesCollection::merge() over the same generations: every file of the merged directory (LUCENE index / hits.data:
except the PFor padding the reference leaves uninitialised) for host-written, device-written and reference-committed generations whose
hits carry payloads, the encoders' payload edges in re-encoded postings, the same bytes as trn_merge_sources when no written hit carries a
payload, the merged segment read back through exec_matches like the reference, and the refusals, each followed by a good call."""
import numpy as np
import pytest

import trinity_b200 as tb
from idxutil import read_dir, term_names
from matchutil import assert_same_matches, gpu_as_list, ref_build
from mergeutil import model_plan, random_specs, ref_merge, stored_hits, write_generation
from payutil import ref_index_payloads, zipf_payloads
from test_merge_model_cpu import SHAPES
from trinity_b200.segments import SegmentCollection

pytestmark = pytest.mark.gpu
G, L = tb.CODEC_GOOGLE, tb.CODEC_LUCENE
OUT = pytest.mark.parametrize("out_codec", [G, L], ids=["google", "lucene"])
DISABLE = pytest.mark.parametrize("disable", [False, True], ids=["opt", "noopt"])


@pytest.fixture(scope="module")
def gpu():
    g = tb.GpuIndexSource(0)
    yield g
    g.close()


def _compare(got_dir, want_dir, codec):
    want, got = read_dir(want_dir), read_dir(got_dir)
    assert sorted(want) == sorted(got)
    for f in want:
        if codec == L and f in ("index", "hits.data"):
            assert got[f].size == want[f].size, f
            diff = np.flatnonzero(got[f] != want[f])
            # the reference leaves the padding of the PFor byte container uninitialised (fastpfor.h:196-198): only there, and only zeros of ours
            assert np.all(got[f][diff] == 0), f"{f} differs at non-padding bytes {diff[:10]}"
        else:
            assert np.array_equal(got[f], want[f]), f


def _against_the_reference(m, tmp_path, paths, out_codec, disable, tag=""):
    ref_fs, _ = ref_merge(out_codec, tmp_path / f"ref{tag}" / "100", paths, disable, m.field_statistics["docsCnt"])
    assert m.field_statistics == ref_fs
    m.write(tmp_path / f"dev{tag}" / "100")
    _compare(tmp_path / f"dev{tag}" / "100", tmp_path / f"ref{tag}" / "100", out_codec)


def _host_sources(root, codecs, seed, max_position=None, **kw):
    specs, updated = random_specs(np.random.default_rng(seed), codecs, **kw)
    if max_position:  # positions scaled into 1..max_position, order kept
        specs = [{n: [(d, [(1 + p * (max_position - 1) // 16383, pl) for p, pl in h]) for d, h in post] for n, post in s.items()} for s in specs]
    paths = [root / f"{g + 1}" for g in range(len(codecs))]
    return paths, [write_generation(p, c, s, u) for p, c, s, u in zip(paths, codecs, specs, updated)], specs


# ------------------------------------------------------------------------------------------------------------------ host-written sources
@pytest.mark.parametrize("shape", list(SHAPES))
@OUT
@DISABLE
def test_host_written_payload_generations(gpu, tmp_path, shape, out_codec, disable):
    """random_specs(payloads=True) generations (the reference encoders' bytes, replaced and erased documents) in every shape of
    test_merge_model_cpu"""
    codecs = SHAPES[shape]
    paths, srcs, _ = _host_sources(tmp_path / "src", codecs, seed=len(shape) * 31 + out_codec, payloads=True)
    m = gpu.merge_sources(out_codec, srcs, disable, payloads=True)
    _against_the_reference(m, tmp_path, paths, out_codec, disable)
    if len(codecs) > 1 or disable or codecs[0] != out_codec:
        assert m.counts["reencoded"] > 0


# ---------------------------------------------------------------------------------------------------------------- device-written sources
def _payload_corpus(rng, docids, nterms, frac):
    lens = rng.integers(1, 40, len(docids))
    w = 1.0 / np.arange(1, nterms + 1)
    tok = rng.choice(nterms, int(lens.sum()), p=w / w.sum()).astype(np.uint32)
    offs = np.r_[0, np.cumsum(lens)].astype(np.uint64)
    plens, pays = zipf_payloads(rng, len(tok))
    plens[rng.random(len(tok)) >= frac] = 0
    return offs, tok, plens, pays


def _device_generations(gpu, root, codecs, ndocs, nterms, seed, frac=0.5):
    """generations indexed by trn_index_documents_payloads, oldest first: each holds docIDs drawn from a range the older ones share (the
    ones an older generation holds are replaced), and erases a few older documents"""
    rng = np.random.default_rng(seed)
    names, live, paths = term_names(nterms), set(), []
    for k, codec in enumerate(codecs):
        docids = rng.permutation(np.unique(rng.integers(1, ndocs * 2, ndocs)).astype(np.uint32))
        offs, tok, plens, pays = _payload_corpus(rng, docids, nterms, frac)
        seg = gpu.index_documents_flat(codec, docids, offs, tok, nterms, None, plens, pays)
        older = np.array(sorted(live), np.uint32)
        replaced, erased = np.intersect1d(docids, older), np.setdiff1d(older[::13], docids)
        p = root / f"{k + 1}"
        seg.write(p, names, replaced=replaced, erased=erased)
        paths.append(p)
        live = (live - set(erased.tolist())) | set(docids.tolist())
    return paths, live


@OUT
@DISABLE
@pytest.mark.parametrize("codecs", [[G, L], [L, G, L], [G, G, L, G]], ids=["GL", "LGL", "GGLG"])
def test_device_written_generations(gpu, tmp_path, out_codec, disable, codecs):
    paths, live = _device_generations(gpu, tmp_path / "src", codecs, 3000, 300, seed=len(codecs) * 5 + out_codec)
    m = SegmentCollection(paths).merge(out_codec, disable, payloads=True)
    assert m.field_statistics["docsCnt"] == len(live)
    assert m.counts["reencoded"] > 0
    _against_the_reference(m, tmp_path, paths, out_codec, disable)


@OUT
def test_reference_committed_generations(gpu, tmp_path, out_codec):
    """generations the reference's own SegmentIndexSession commits with payloads (shared docIDs, no registries)"""
    rng = np.random.default_rng(23 + out_codec)
    names, paths = term_names(200), []
    for k, codec in enumerate([L, G, L]):
        docids = np.unique(rng.integers(1, 5000, 2500)).astype(np.uint32)
        offs, tok, plens, pays = _payload_corpus(rng, docids, len(names), 0.7)
        p = tmp_path / "src" / f"{k + 1}"
        ref_index_payloads(codec, p, names, docids, offs, tok, None, plens, pays)
        paths.append(p)
    m = SegmentCollection(paths).merge(out_codec, False, payloads=True)
    assert m.counts["reencoded"] > 0
    _against_the_reference(m, tmp_path, paths, out_codec, False)


# ----------------------------------------------------------------------------------------------------------------------------- edges
def _pl(rng, n):
    return bytes(rng.integers(0, 256, n, dtype=np.uint8))


def _doc(rng, d, sizes, positions=None):
    ps = sorted(int(p) for p in rng.integers(1, 16384, len(sizes))) if positions is None else list(positions)
    return (int(d), [(p, _pl(rng, int(s))) for p, s in zip(ps, sizes)])


def _docids(rng, n, first=1, gap=40):
    return [int(x) for x in first + np.cumsum(rng.integers(1, gap, n))]


def _edge_terms(kind, rng):
    """{name: postings} of the older generation: one edge of the encoders' payload handling per kind"""
    if kind == "sizes":  # every size 0..8, in every order inside a document
        return {"e": [_doc(rng, d, [(i + k) % 9 for k in range(9)]) for i, d in enumerate(_docids(rng, 60))]}
    if kind == "changes":  # the size changes at every hit, at document starts only, never
        return {"every": [_doc(rng, d, [1 + (k % 2) * 6 for k in range(4)]) for d in _docids(rng, 70)],
                "starts": [_doc(rng, d, [1 + i % 8] * (1 + i % 4)) for i, d in enumerate(_docids(rng, 70))],
                "never": [_doc(rng, d, [5] * (1 + i % 3)) for i, d in enumerate(_docids(rng, 70))]}
    if kind == "pos0":  # a document's first hit at position 0 with a payload
        out = []
        for i, d in enumerate(_docids(rng, 150)):
            n = 1 + i % 4
            out.append(_doc(rng, d, [1 + i % 8] + [(i + k) % 9 for k in range(1, n)], [0] + sorted(int(p) for p in rng.integers(1, 16384, n - 1))))
        return {"zero": out}
    if kind == "shorter":  # GOOGLE: a shorter payload after a longer one (its reader keeps the longer one's high bytes)
        return {"s": [_doc(rng, d, [8, 2, 5, 1, 8, 0, 3, 7, 1]) for d in _docids(rng, 50)]}
    if kind == "long":  # a 17 000-hit document whose size changes at random
        long = (500, [(p, _pl(rng, int(s))) for p, s in zip(np.sort(rng.integers(1, 16384, 17000)).tolist(), rng.integers(0, 9, 17000))])
        return {"l": [_doc(rng, d, [3, 0]) for d in _docids(rng, 10)] + [long] + [_doc(rng, d, [1]) for d in _docids(rng, 10, 600)]}
    if kind == "blocks":  # full 128-hit blocks, every PFor form of the size int-block; documents spanning blocks
        few8 = lambda i, k: 8 if (i * 3 + k) % 41 == 0 else 0  # noqa: E731
        forms = {"all0": lambda i, k: 0, "all3": lambda i, k: 3, "few8": few8, "mixed": lambda i, k: (i * 7 + k * 3) % 9}
        out = {n: [_doc(rng, d, [f(i, k) for k in range(3)]) for i, d in enumerate(_docids(rng, 300))] for n, f in forms.items()}
        out["span"] = [_doc(rng, d, [(k // 20) % 9 for k in range(50 + 37 * i)]) for i, d in enumerate(_docids(rng, 8))]
        return out
    if kind == "five":  # docID deltas of 2^28 and more: 5-byte varbyte codes
        return {"v": [_doc(rng, d, [i % 9, 8]) for i, d in enumerate([7, 7 + (1 << 28) + 3, 7 + (1 << 29), 4_000_000_000])]}
    if kind == "high":  # docIDs up to 2^32 - 2
        return {"h": [_doc(rng, d, [1 + i % 8, i % 9]) for i, d in enumerate(sorted(2**32 - 2 - 7 * np.arange(200)))]}
    raise KeyError(kind)


EDGES = ["sizes", "changes", "pos0", "shorter", "long", "blocks", "five", "high"]


@pytest.mark.parametrize("kind", EDGES)
@pytest.mark.parametrize("src_codec", [G, L], ids=["from-google", "from-lucene"])
@OUT
def test_edges(gpu, tmp_path, kind, src_codec, out_codec):
    """the older generation holds the edge terms; the newer one holds every third of their documents (so its postings win) and lists
    every fifth as updated (so they are masked): the written postings of the older one sit between postings that are not written, in
    the same GOOGLE block and LUCENE 128-hit block"""
    rng = np.random.default_rng(EDGES.index(kind) * 4 + src_codec * 2 + out_codec)
    old = _edge_terms(kind, rng)
    new, updated = {}, set()
    for n, post in old.items():
        new[n] = [_doc(rng, d, [int(s) for s in rng.integers(0, 9, 2)]) for d, _ in post[::3]]
        if kind != "high":  # the reference's registry does not find docIDs this close to 2^32: only the newer holder decides there
            updated |= {d for d, _ in post[1::5]}
    new["zz"] = [_doc(rng, 3, [2])]
    paths = [tmp_path / "src" / "1", tmp_path / "src" / "2"]
    srcs = [write_generation(paths[0], src_codec, old), write_generation(paths[1], src_codec, new, sorted(updated))]
    m = gpu.merge_sources(out_codec, srcs, False, payloads=True)
    assert m.counts["appended"] == (1 if src_codec == out_codec else 0) and m.counts["reencoded"] == len(new) - m.counts["appended"]
    _against_the_reference(m, tmp_path, paths, out_codec, False)


# ------------------------------------------------------------------------------------------------------------- no payloads, same bytes
def _same_result(a, b):
    assert np.array_equal(a.index, b.index) and np.array_equal(a.hits, b.hits) and np.array_equal(a.terms, b.terms)
    assert a.names == b.names and a.field_statistics == b.field_statistics and a.counts == b.counts


@OUT
@pytest.mark.parametrize("kind", ["no-payloads", "all-sizes-0"])
def test_without_payloads_both_entry_points_agree(gpu, tmp_path, out_codec, kind):
    if kind == "no-payloads":
        _, srcs, _ = _host_sources(tmp_path / "src", [G, L, G], seed=7 + out_codec)
    else:  # device-indexed with a payload array whose sizes are all 0
        paths, _ = _device_generations(gpu, tmp_path / "src", [L, G, L], 2000, 150, seed=3 + out_codec, frac=0.0)
        coll = SegmentCollection(paths)
        srcs = [tb.MergeSource.of_segment(s, p, g) for s, p, g in zip(coll.segments, coll.paths, coll.generations)]
    for disable in (False, True):
        a = gpu.merge_sources(out_codec, srcs, disable)
        b = gpu.merge_sources(out_codec, srcs, disable, payloads=True)
        assert a.counts["reencoded"] > 0
        _same_result(a, b)


# ------------------------------------------------------------------------------------------------------------------- reading it back
def _merged_postings(srcs, specs):
    """merge() over the specs: per name, of every docID the newest holder's stored hits unless a newer registry masks it"""
    plan = model_plan(G, srcs, False)
    upd = dict(zip(plan["upd_docid"], plan["upd_first"]))
    out = {}
    for nm in sorted({n for s in specs for n in s}, key=str.encode):
        post = {}
        for j, s in enumerate(plan["order"]):
            for d, hits in specs[s].get(nm, []):
                if d not in post:
                    post[d] = None if (d in upd and upd[d] < j) else stored_hits(hits)
        out[nm] = [(d, h) for d, h in sorted(post.items()) if h is not None]
    return out


def _as_list(post):
    docs = np.array([d for d, _ in post], np.uint32)
    freqs = np.array([len(h) for _, h in post], np.uint32)
    hits = [x for _, h in post for x in h]
    pos = np.array([p for p, _ in hits], np.uint32)
    sz = np.array([len(b) for _, b in hits], np.uint8)
    pv = np.array([int.from_bytes(b, "little") for _, b in hits], np.uint64)
    return docs, freqs, pos, sz, pv


@OUT
def test_merged_payloads_read_back_like_the_reference(gpu, tmp_path, out_codec):
    """exec_matches over the uploaded merge: the matched terms and every hit with its payload == the reference's exec over the merged
    postings (bytes equal to its merged directory's, checked first)"""
    codecs = [G, L, G]
    # positions below 8192: the reference's exec_query keeps a document's hits in a DocWordsSpace of max_indexed_position() = 8192
    paths, srcs, specs = _host_sources(tmp_path / "src", codecs, seed=77 + out_codec, max_position=8000, payloads=True)
    m = gpu.merge_sources(out_codec, srcs, False, payloads=True)
    _against_the_reference(m, tmp_path, paths, out_codec, False)
    merged = _merged_postings(srcs, specs)
    assert m.names == [n for n in merged if merged[n]]
    lists = [_as_list(merged[n]) for n in m.names]
    maxdoc = max(int(l[0].max()) for l in lists)
    r = ref_build(out_codec, lists, m.names, maxdoc)
    g = tb.GpuIndexSource(0)
    try:
        g.upload(out_codec, m.index, m.terms, maxdoc)
        if out_codec == L:
            g.upload_hits(m.index, m.hits)
        td = tb.TermDictionary(m.names)
        top = sorted(m.names, key=lambda n: -len(merged[n]))[:6]
        qs = [top[0], top[1], f"{top[0]} AND {top[1]}", f"{top[2]} OR {top[3]} OR {top[4]}", f"{top[1]} NOT {top[5]}"]
        qs += ["a OR ab OR abc"] if {"a", "ab", "abc"} <= set(m.names) else []
        res = g.exec_matches([tb.parse_query(q, td) for q in qs])
        for i, q in enumerate(qs):
            assert_same_matches(gpu_as_list(res, i), r.exec(q), f"out codec {out_codec} [{q}]")
    finally:
        g.close()


# --------------------------------------------------------------------------------------------------------------------------- refusals
def test_refusals_name_the_source_and_term(gpu, tmp_path):
    """a hit above 16383 and one at position 0 without a payload (TRN_ERR_UNSUPPORTED), a stored payload length of 9 (TRN_ERR_FORMAT),
    each in a re-encoded posting; after each, a good call on the same context gives the earlier result"""
    _, good, _ = _host_sources(tmp_path / "good", [G, L], seed=5, payloads=True)
    first = gpu.merge_sources(L, good, False, payloads=True)

    def still_good():
        again = gpu.merge_sources(L, good, False, payloads=True)
        assert np.array_equal(again.index, first.index) and np.array_equal(again.hits, first.hits) and again.names == first.names

    with pytest.raises(tb.TrinityError, match=r"rc=-1: trn_merge_sources_payloads: sources \d and \d share generation"):  # the planner's
        gpu.merge_sources(L, [good[0], good[0]], payloads=True)
    still_good()
    for codec in (G, L):
        src = write_generation(tmp_path / f"high{codec}" / "7", codec, {"a": [(1, [(3, b"x")])], "high": [(5, [(2, b"ab"), (20000, b"")])]})
        with pytest.raises(tb.TrinityError, match=r"rc=-7: trn_merge_sources_payloads: source 0 \(generation 7\), term \[high\]: a hit at position 0 "
                                                  r"without a payload, or above 16383"):
            gpu.merge_sources(G, [src], True, payloads=True)
        still_good()
    # LUCENE: a one-hit tail is varbyte(delta << 1 | changed), the size byte, then the payload bytes; its size byte rewritten
    src = write_generation(tmp_path / "zero" / "7", L, {"a": [(1, [(3, b"")])], "zero": [(5, [(0, b"\xab")])]})
    t = src.terms[list(src.names).index("zero")]
    hdo = int(src.index[t["chunk_off"]:t["chunk_off"] + 4].view("<u4")[0])
    assert src.hits[hdo:hdo + 3].tolist() == [1, 1, 0xAB]
    for size, rc, msg in ((0, -7, "a hit at position 0 without a payload"), (9, -3, "a hit stores a payload of more than 8 bytes")):
        hits = src.hits.copy()
        hits[hdo + 1] = size
        bad = tb.MergeSource(L, 7, src.index, src.terms, src.names, hits)
        with pytest.raises(tb.TrinityError, match=rf"rc={rc}: trn_merge_sources_payloads: source 0 \(generation 7\), term \[zero\]: {msg}"):
            gpu.merge_sources(L, [bad], True, payloads=True)
        still_good()
    # the position-0 hit with its payload is written by the payload entry point and refused by the other
    m = gpu.merge_sources(G, [src], True, payloads=True)
    assert m.field_statistics["sumTermHits"] == 2
    with pytest.raises(tb.TrinityError, match=r"rc=-7: trn_merge_sources: source 0 \(generation 7\), term \[zero\]: a hit with a payload"):
        gpu.merge_sources(G, [src], True)
    still_good()
