"""Shared by the merge tests: the reference's MergeCandidatesCollection behind a C ABI (oracle/_ref/libtrinity_ref_merge.so,
oracle/ref_merge.cpp), a Python restatement of merge()'s term loop, and generations written by the reference's SegmentIndexSession.
TEST INFRASTRUCTURE ONLY — never imported by the product package."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
SO = ROOT / "oracle" / "_ref" / "libtrinity_ref_merge.so"
_lib = None


def load_merge():
    global _lib
    if _lib is None:
        if not SO.exists():
            subprocess.check_call(["bash", str(ROOT / "oracle" / "build_merge.sh")])
        L = C.CDLL(str(SO))
        L.tmrg_last_error.restype = C.c_char_p
        L.tmrg_last_ms.restype = C.c_double
        L.tref_merge.argtypes = [C.c_int, C.c_char_p, C.c_void_p, C.c_uint32, C.c_int, C.c_uint32, C.c_void_p]
        L.tref_consider_tracked_sources.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def ref_merge(out_codec, out_dir, src_dirs, disable_optimizations, docs_cnt):
    """the reference's commit() + merge() of the segment directories into out_dir; returns (field statistics, host ms)"""
    L = load_merge()
    Path(out_dir).mkdir(parents=True, exist_ok=True)
    enc = [str(d).encode() for d in src_dirs]
    arr = (C.c_char_p * max(1, len(enc)))(*enc)
    st = np.zeros(4, np.uint64)
    rc = L.tref_merge(out_codec, str(out_dir).encode(), C.cast(arr, C.c_void_p), len(enc), int(bool(disable_optimizations)), docs_cnt,
                      st.ctypes.data_as(C.c_void_p))
    if rc != 0:
        raise RuntimeError(L.tmrg_last_error().decode())
    return {"sumTermHits": int(st[0]), "totalTerms": int(st[1]), "sumTermsDocs": int(st[2]), "docsCnt": int(st[3])}, float(L.tmrg_last_ms())


def ref_consider_tracked_sources(cands, tracked):
    L = load_merge()
    c, t = np.asarray(cands, np.uint64), np.asarray(tracked, np.uint64)
    g, r = np.zeros(max(1, len(t)), np.uint64), np.zeros(max(1, len(t)), np.uint8)
    L.tref_consider_tracked_sources(c.ctypes.data_as(C.c_void_p), len(c), t.ctypes.data_as(C.c_void_p), len(t), g.ctypes.data_as(C.c_void_p),
                                    r.ctypes.data_as(C.c_void_p))
    return list(zip(g[:len(t)].tolist(), r[:len(t)].tolist()))


def model_plan(out_codec, sources, disable):
    """merge.cpp:6-35 and 127-395 restated over names and tuples: candidate order, output terms (route, stats flag, participants)"""
    order = sorted(range(len(sources)), key=lambda s: -sources[s].generation)
    gens = [sources[s].generation for s in order]
    if len(set(gens)) != len(gens):
        raise ValueError("equal generations")
    updaters_before = np.cumsum([0] + [1 if (sources[s].updated_docids is not None and len(sources[s].updated_docids)) else 0 for s in order])
    key = lambda n: n.encode() if isinstance(n, str) else n
    allnames = sorted({key(n) for m in sources for n in m.names})
    pos = [{key(n): i for i, n in enumerate(sources[s].names)} for s in order]
    route, stats, parts = [], [], []
    for nm in allnames:
        holders = [j for j in range(len(order)) if nm in pos[j]]
        docs = lambda j: int(sources[order[j]].terms[pos[j][nm]]["documents"])
        with_docs = [(j, pos[j][nm]) for j in holders if docs(j)]
        if not with_docs:
            continue
        if len(holders) == 1:
            j = holders[0]
            app = sources[order[j]].codec == out_codec and updaters_before[j] == 0 and not disable
            route.append(0 if app else 1)
            stats.append(0 if app else 1)
        else:
            same = all(sources[order[j]].codec == out_codec for j in holders)
            route.append(1)
            stats.append(0 if (same and not disable) else 1)
        parts.append(with_docs)
    u = {}
    for j, s in enumerate(order):
        for d in (sources[s].updated_docids if sources[s].updated_docids is not None else []):
            u.setdefault(int(d), j)
    ud = sorted(u)
    return {"order": order, "route": route, "stats": stats, "parts": parts, "upd_docid": ud, "upd_first": [u[d] for d in ud]}


# ---------------------------------------------------------------------------------------------------------------- host-built sources
# A generation is {name: [(docID, [(position, payload bytes), ...]), ...]} (docIDs ascending) plus its codec, generation number and updated
# docIDs.  It is encoded with the host IndexBuilder (the reference encoders' bytes) and written with segment_write, which the reference's
# SegmentIndexSource opens; the model below merges the same postings the way merge.cpp does and encodes them with a host IndexBuilder.

def _key(n):
    return n.encode() if isinstance(n, str) else n


def stored_hits(hits):
    """what the encoders store of a document's hits: a hit at position 0 without a payload is dropped (google_codec.cpp, lucene_codec.cpp)"""
    return [(p, pl) for p, pl in hits if p or pl]


def _encode_term(b, postings):
    b.begin_term()
    for d, hits in postings:
        b.begin_document(int(d))
        for p, pl in hits:
            b.new_hit(int(p), pl)
        b.end_document()
    return b.end_term()


def write_generation(path, codec, spec, updated=()):
    """encodes spec with the host IndexBuilder and writes the segment directory; returns the MergeSource of it"""
    import trinity_b200 as tb
    from trinity_b200._ffi import TERM_DTYPE

    names = sorted(spec, key=_key)
    b = tb.IndexBuilder(codec)
    terms = np.array([_encode_term(b, spec[n]) for n in names], TERM_DTYPE)
    index, hits = b.index(), b.hits()
    docs = {d for n in names for d, _ in spec[n]}
    fs = {"sumTermHits": sum(len(h) for n in names for _, h in spec[n]), "totalTerms": len(names),
          "sumTermsDocs": sum(len(spec[n]) for n in names), "docsCnt": len(docs)}
    tb.segment_write(path, codec, index, hits if codec == tb.CODEC_LUCENE else None, terms, names, fs, sorted(set(int(u) for u in updated)))
    return tb.MergeSource(codec, int(Path(path).name), index, terms, names, hits if codec == tb.CODEC_LUCENE else None,
                          np.asarray(sorted(set(int(u) for u in updated)), np.uint32))


def model_merge(out_codec, sources, specs, disable):
    """merge.cpp over host-built sources: (index, hits, terms, names, field statistics).  specs[i] = the postings of sources[i]."""
    import trinity_b200 as tb
    from trinity_b200._ffi import TERM_DTYPE

    plan = model_plan(out_codec, sources, disable)
    order = plan["order"]
    upd = dict(zip(plan["upd_docid"], plan["upd_first"]))
    lucene = out_codec == tb.CODEC_LUCENE
    b = tb.IndexBuilder(out_codec)
    enc = []  # per output term: the builder's tuple of a re-encoded term, or None
    written, fs = [], {"sumTermHits": 0, "totalTerms": 0, "sumTermsDocs": 0, "docsCnt": 0}
    for route, stats, parts in zip(plan["route"], plan["stats"], plan["parts"]):
        j0, t0 = parts[0]
        nm = sources[order[j0]].names[t0]
        if route == 0:
            enc.append(None)
            written.append([d for d, _ in specs[order[j0]][nm]])
            continue
        post = {}
        for j, t in parts:  # newest first: the first holder of a docID decides
            for d, hits in specs[order[j]][sources[order[j]].names[t]]:
                if d not in post:
                    post[d] = None if (d in upd and upd[d] < j) else stored_hits(hits)
        out = [(d, h) for d, h in sorted(post.items()) if h is not None]
        enc.append(_encode_term(b, out))
        written.append([d for d, _ in out])
        if stats:
            fs["sumTermsDocs"] += len(out)
            fs["sumTermHits"] += sum(len(h) for _, h in out)
    bi, bh = b.index(), b.hits()
    index, hits, terms, names = [], [], [], []
    io = ho = 0
    for e, parts, docs in zip(enc, plan["parts"], written):
        j0, t0 = parts[0]
        s = sources[order[j0]]
        if e is None:
            t = s.terms[t0]
            chunk, src_hits = s.index[t["chunk_off"]:t["chunk_off"] + t["chunk_len"]].copy(), s.hits
        else:
            chunk, src_hits = bi[e[1]:e[1] + e[2]].copy(), bh
        if lucene:
            hdo, pcs = int(chunk[:4].view("<u4")[0]), int(chunk[8:12].view("<u4")[0])
            hits.append(src_hits[hdo:hdo + pcs])
            chunk[:4] = np.frombuffer(np.uint32(ho).tobytes(), np.uint8)
            ho += pcs
        index.append(chunk)
        if docs:
            terms.append((len(docs), io, len(chunk)))
            names.append(s.names[t0])
        io += len(chunk)
    fs["totalTerms"] = len(terms)
    fs["docsCnt"] = len({d for docs in written for d in docs})
    cat = lambda v: np.concatenate(v).astype(np.uint8) if v else np.zeros(0, np.uint8)
    return cat(index), cat(hits), np.array(terms, TERM_DTYPE), names, fs


def random_specs(rng, codecs, ndocs=300, payloads=False, freq0=False):
    """generations oldest first: shared and unique terms (prefixes of each other, more than 64 of them), lists of 1 to ~10 blocks, newer
    generations replacing and erasing older documents, one term every posting of which is masked (an orphan when re-encoded)"""
    names = ["a", "ab", "abc", "b", "ba"] + [f"t{i:03d}" for i in range(80)]
    specs, updated, live = [], [], set()
    for g, codec in enumerate(codecs):
        docs = sorted(int(d) for d in rng.choice(ndocs * 3, ndocs, replace=False) + 1)
        older = sorted(live)
        upd = set(int(d) for d in rng.choice(older, min(len(older), ndocs // 3), replace=False)) if older else set()
        spec = {}
        for n in rng.choice(names, int(rng.integers(20, len(names))), replace=False):
            k = int(rng.integers(1, ndocs))
            sel = sorted(int(d) for d in rng.choice(docs, k, replace=False))
            post = []
            for d in sel:
                f = int(rng.integers(0 if (freq0 and codec == 1) else 1, 5))
                ps = sorted(int(p) for p in rng.integers(1, 16384, f))
                pl = [bytes(rng.integers(0, 256, int(rng.integers(1, 5)), dtype=np.uint8)) if payloads and rng.random() < 0.3 else b"" for _ in ps]
                post.append((d, list(zip(ps, pl))))
            spec[str(n)] = post
        if g == 0:
            spec["orphan"] = [(d, [(1, b"")]) for d in docs[:40]]
        elif g == 1:
            upd |= set(docs[:40]) if False else set(d for d, _ in specs[0]["orphan"])
        specs.append(spec)
        updated.append(sorted(upd))
        live |= set(docs)
    return specs, updated
