"""Query-token intersections (test infrastructure): two Python transcriptions of what Trinity::intersect_impl computes — the sequential
state machine of the reference (ctx::consider, intersect.cpp:53-100, line by line) and the epoch restatement the device passes implement
(DESIGN.md §4, csrc/isectplan.h) — and the ctypes wrapper of the reference oracle (oracle/_ref/libtrinity_ref_isect.so)."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ISECT_SO = ROOT / "oracle" / "_ref" / "libtrinity_ref_isect.so"


# ------------------------------------------------------------------------------------------------ the considered stream
def considered_stream(group_docs, masked=(), orig_mask=None):
    """[(docID, mask)] of the considered documents in docID order: group_docs[g] = the docIDs of group g (the union of its known tokens'
    postings); orig_mask defaults to the mask of the groups with a known token (pass 0 when a token is unknown)"""
    if orig_mask is None:
        orig_mask = 0
        for g, d in enumerate(group_docs):
            if len(d):
                orig_mask |= 1 << g
    masks = {}
    for g, d in enumerate(group_docs):
        for x in d:
            masks[int(x)] = masks.get(int(x), 0) | (1 << g)
    mk = set(int(x) for x in masked)
    return [(d, m) for d, m in sorted(masks.items()) if m != orig_mask and d not in mk]


# ------------------------------------------------------------------------------------------------ sequential transcription
def consider_sequential(masks, index_wrap=255):
    """ctx::consider over the considered masks, line by line (indexPrev is a uint8_t: index_wrap = 255) -> {mask: cnt}; index_wrap = None
    models an index that does not wrap, which the tests use to show that a case reaches the wrap"""
    matches = []  # [[v, cnt]]
    map_prev, index_prev = 0, 0
    wrap = (lambda i: i) if index_wrap is None else (lambda i: i & index_wrap)
    for m in masks:
        if m == map_prev:
            matches[index_prev][1] += 1
            continue
        n = len(matches)
        map_prev = m
        i = 0
        absorbed = False
        while i < n:
            v = matches[i][0]
            if (v & m) == m:
                if m == v:
                    matches[i][1] += 1
                index_prev = wrap(i)
                absorbed = True
                break
            elif (m & v) == v:
                matches[i] = matches[-1]
                matches.pop()
                n -= 1
            else:
                i += 1
        if not absorbed:
            index_prev = wrap(n)
            matches.append([m, 1])
    return {v: c for v, c in matches}


# ------------------------------------------------------------------------------------------------ epoch restatement
def epoch_plan(masks, firsts):
    """the host step: (epoch starts, epoch arrays as [(mask, final index or -1)], final antichain) from the distinct masks and their
    first docIDs"""
    arr, starts, snaps = [], [], []
    for f, m in sorted(zip(firsts, masks)):
        i, absorbed = 0, False
        while i < len(arr):
            v = arr[i]
            if (v & m) == m:
                absorbed = True
                break
            elif (m & v) == v:
                arr[i] = arr[-1]
                arr.pop()
            else:
                i += 1
        if absorbed:
            continue
        arr.append(m)
        starts.append(f)
        snaps.append(list(arr))
    slot = {v: i for i, v in enumerate(arr)}
    return starts, [[(v, slot.get(v, -1)) for v in s] for s in snaps], list(arr)


def consider_epochs(stream):
    """the restatement over [(docID, mask)]: every document adds to the entry its epoch's array gives it, on its own -> {mask: cnt}"""
    import bisect
    first = {}
    for d, m in stream:
        first.setdefault(m, d)
    starts, arrays, final = epoch_plan(list(first), list(first.values()))
    counts = [0] * len(final)
    prev = 0
    for d, m in stream:
        arr = arrays[bisect.bisect_right(starts, d) - 1]
        i = next(k for k, (v, _) in enumerate(arr) if (v & m) == m)
        if prev == m:
            s = arr[i & 255][1]  # a run goes on: matches[indexPrev], indexPrev a uint8_t
        elif arr[i][0] == m:
            s = arr[i][1]
        else:
            s = -1  # the first document of a run a strict superset absorbs is not counted
        if s >= 0:
            counts[s] += 1
        prev = m
    return dict(zip(final, counts))


def finalize_order(pairs):
    """the device's deterministic refinement of finalize()'s order: popcount desc, count desc, mask asc"""
    return sorted(pairs, key=lambda p: (-bin(p[0]).count("1"), -p[1], p[0]))


# ------------------------------------------------------------------------------------------------ the reference oracle
def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class RefIsect:
    def __init__(self):
        if not ISECT_SO.exists():
            subprocess.check_call(["bash", str(ROOT / "oracle" / "build_intersect.sh")])
        L = self.L = C.CDLL(str(ISECT_SO))
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.tisect_last_error.restype = C.c_char_p
        L.tisect_source.restype = vp
        L.tisect_source.argtypes = [C.c_int, vp, u64, vp, u64, vp, vp, vp, vp, u32]
        L.tisect_collection.restype = vp
        L.tisect_collection.argtypes = [vp, u32]
        L.tisect_free.argtypes = [vp]
        L.tisect_run.restype = C.c_int64
        L.tisect_run.argtypes = [vp, u32, vp, vp, vp, u32]
        L.tisect_run_collection.restype = C.c_int64
        L.tisect_run_collection.argtypes = [vp, u32, vp, vp]
        L.tisect_last.argtypes = [vp, vp, vp]

    def source(self, codec, index, names, terms, hits=None):
        """an in-memory IndexSource over index bytes (either codec; LUCENE: and its hits.data) and its terms"""
        index = np.ascontiguousarray(index, np.uint8)
        hits = np.ascontiguousarray(hits if hits is not None else np.zeros(0), np.uint8)
        enc = [n.encode() for n in names]
        arr = (C.c_char_p * len(enc))(*enc)
        cols = [np.ascontiguousarray(terms[f], np.uint32) for f in ("documents", "chunk_off", "chunk_len")]
        h = self.L.tisect_source(codec, _p(index), index.size, _p(hits) if hits.size else None, hits.size, C.cast(arr, C.c_void_p), *[_p(c) for c in cols], len(enc))
        if not h:
            raise RuntimeError(self.L.tisect_last_error().decode())
        return _Handle(self, h)

    def collection(self, dirs):
        enc = [str(p).encode() for p in dirs]
        arr = (C.c_char_p * len(enc))(*enc)
        h = self.L.tisect_collection(C.cast(arr, C.c_void_p), len(enc))
        if not h:
            raise RuntimeError(self.L.tisect_last_error().decode())
        return _Handle(self, h)


class _Handle:
    def __init__(self, rl, h):
        self.rl, self.h = rl, C.c_void_p(h)

    def _groups(self, token_groups):
        offs = np.ascontiguousarray(np.concatenate([[0], np.cumsum([len(g) for g in token_groups])]), np.uint32)
        enc = [t.encode() for g in token_groups for t in g] or [b""]
        return offs, (C.c_char_p * len(enc))(*enc)

    def _last(self, n):
        if n < 0:
            raise RuntimeError(self.rl.L.tisect_last_error().decode())
        m, c = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint32)
        self.rl.L.tisect_last(self.h, _p(m), _p(c))
        return [(int(m[i]), int(c[i])) for i in range(n)]

    def intersect(self, token_groups, masked=()):
        """intersect(0, tokens, src, registry holding `masked`) -> [(mask, count)] in the reference's (finalize) order"""
        offs, names = self._groups(token_groups)
        mk = np.ascontiguousarray(masked, np.uint32)
        return self._last(self.rl.L.tisect_run(self.h, len(token_groups), _p(offs), C.cast(names, C.c_void_p), _p(mk), len(mk)))

    def intersect_collection(self, token_groups):
        """intersect(0, tokens, collection) -> [(mask, count)] by mask"""
        offs, names = self._groups(token_groups)
        return self._last(self.rl.L.tisect_run_collection(self.h, len(token_groups), _p(offs), C.cast(names, C.c_void_p)))

    def __del__(self):
        try:
            self.rl.L.tisect_free(self.h)
        except Exception:
            pass
