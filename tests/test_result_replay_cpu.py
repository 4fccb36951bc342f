"""trn_result_for_each / trn_result_decode (the consider(docid_t) replay of a result, matches.h:149-171) over hand-built results in both
forms: plain docIDs and the compact segments of TRN_MODE_DOCS_COMPACT (docIDs / 16-bit offsets / bucketed 8-bit offsets / tile bitmaps).
No GPU involved."""
import ctypes as C

import numpy as np
import pytest

import trinity_b200 as tb
from trinity_b200._ffi import CONSIDER_FN, TrnResult, lib

ENC_U32, ENC_U16, ENC_BITMAP, ENC_U8B = 0, 1, 2, 3


def _compact(queries, shift):
    """queries: list of (tile_lo, [docid arrays per item], [encodings]) -> TrnResult + the arrays that back it"""
    words, desc, qitems, offsets = [], [], [], [0]
    for tile_lo, items, encs in queries:
        base_item = len(desc)
        for j, (ids, enc) in enumerate(zip(items, encs)):
            ids = np.asarray(ids, np.uint32)
            first = (tile_lo + j) << shift
            if len(ids) == 0:
                desc.append(0)
                continue
            desc.append(len(ids) | (enc << 30))
            if enc == ENC_U32:
                words += [int(x) for x in ids]
            elif enc == ENC_U16:
                rel = (ids - first).astype(np.uint32)
                assert rel.max() < (1 << shift)
                if len(rel) & 1:
                    rel = np.append(rel, 0)
                words += [int(rel[i]) | (int(rel[i + 1]) << 16) for i in range(0, len(rel), 2)]
            elif enc == ENC_U8B:
                rel = (ids - first).astype(np.uint32)
                nbk = (1 << shift) >> 8
                cnt = np.bincount(rel >> 8, minlength=nbk).astype(np.uint8)
                assert np.bincount(rel >> 8, minlength=nbk).max() < 256
                by = np.concatenate([cnt, (rel & 255).astype(np.uint8)])
                by = np.concatenate([by, np.zeros((-len(by)) % 4, np.uint8)])
                words += [int(x) for x in by.view(np.uint32)]
            else:
                bm = np.zeros((1 << shift) // 32, np.uint32)
                rel = ids - first
                np.bitwise_or.at(bm, rel >> 5, np.uint32(1) << (rel & 31).astype(np.uint32))
                words += [int(x) for x in bm]
        qitems.append((base_item, len(items), tile_lo, shift))
        offsets.append(len(words))
    w = np.asarray(words if words else [0], np.uint32)
    d = np.asarray(desc if desc else [0], np.uint32)
    qi = np.asarray(qitems, np.uint32).reshape(-1, 4)
    off = np.asarray(offsets, np.uint64)
    counts = np.asarray([sum(len(x) for x in q[1]) for q in queries], np.uint64)
    r = TrnResult()
    r.nq = len(queries)
    r.offsets = off.ctypes.data_as(C.POINTER(C.c_uint64))
    r.words = w.ctypes.data_as(C.POINTER(C.c_uint32))
    r.total_words = len(words)
    r.item_desc = d.ctypes.data_as(C.POINTER(C.c_uint32))
    r.qitems = qi.ctypes.data_as(C.c_void_p)
    r.match_counts = counts.ctypes.data_as(C.POINTER(C.c_uint64))
    return r, (w, d, qi, off, counts)


def _decode(r, q, cap):
    out = np.zeros(max(cap, 1), np.uint32)
    n = C.c_uint64()
    rc = lib().trn_result_decode(C.byref(r), q, out.ctypes.data_as(C.c_void_p), cap, C.byref(n))
    return rc, int(n.value), out[: min(cap, int(n.value))]


def test_compact_segments_replay_in_every_encoding():
    shift = 12
    rng = np.random.default_rng(3)

    def tile(j, n):
        return np.sort(rng.choice(1 << shift, size=n, replace=False).astype(np.uint32)) + np.uint32(j << shift)

    q0 = (5, [tile(5, 7), np.zeros(0, np.uint32), tile(7, 900), tile(8, 1), tile(9, 4096)], [ENC_U16, ENC_U16, ENC_BITMAP, ENC_U16, ENC_BITMAP])
    q1 = (0, [np.array([3, 9, 70000, 4000000000], np.uint32), np.array([4000000001], np.uint32)], [ENC_U32, ENC_U32])  # lead-block groups: any docIDs
    q2 = (0, [], [])
    q3 = (1 << 19, [tile(1 << 19, 33)], [ENC_U16])  # a tile high up in the docID space
    # bucketed 8-bit offsets: buckets with 0, 1 and many documents, a count that is not a multiple of 4 (pad bytes), next to other forms
    q4 = (40, [tile(40, 301), tile(41, 5), tile(42, 2000), tile(43, 64)], [ENC_U8B, ENC_U8B, ENC_BITMAP, ENC_U8B])
    r, keep = _compact([q0, q1, q2, q3, q4], shift)
    for q, (lo, items, _) in enumerate([q0, q1, q2, q3, q4]):
        want = np.concatenate([np.asarray(x, np.uint32) for x in items]) if items else np.zeros(0, np.uint32)
        rc, n, got = _decode(r, q, len(want) + 3)
        assert rc == 0 and n == len(want) and np.array_equal(got, want), q
        seen = []
        fn = CONSIDER_FN(lambda ctx, d: seen.append(d) or 0)
        assert lib().trn_result_for_each(C.byref(r), q, fn, None) == 0
        assert seen == [int(x) for x in want]
    # capacity: the count is still reported
    rc, n, _ = _decode(r, 0, 5)
    assert rc == -6 and n == 7 + 900 + 1 + 4096
    # a consumer that stops the replay (aborted_search_exception in the reference)
    seen = []
    fn = CONSIDER_FN(lambda ctx, d: (seen.append(d), 1 if len(seen) == 10 else 0)[1])
    assert lib().trn_result_for_each(C.byref(r), 0, fn, None) == 0 and len(seen) == 10


@pytest.mark.parametrize("shift", [13, 14])
def test_compact_segments_of_the_last_tile_below_2_32(shift):
    """the tile base of the last tile of the docID space: (tile_lo << tile_shift) + offset must reach 2^32 - 2 without wrapping"""
    top = 2**32 - 2  # largest valid docID (DocIDsEND = 2^32 - 1)
    tile_lo = (2**32 >> shift) - 1
    first = tile_lo << shift
    ids = np.array([first, first + 1, first + 255, first + 256, first + (1 << shift) // 2, top - 1, top], np.uint32)
    qs = [(tile_lo, [ids], [enc]) for enc in (ENC_U16, ENC_U8B, ENC_BITMAP)]
    # and one query whose last item is the top tile, behind the tile below it
    below = ids - np.uint32(1 << shift)
    qs.append((tile_lo - 1, [below, ids], [ENC_U8B, ENC_U16]))
    r, keep = _compact(qs, shift)
    for q, (_, items, _) in enumerate(qs):
        want = np.concatenate(items)
        rc, n, got = _decode(r, q, len(want))
        assert rc == 0 and n == len(want) and np.array_equal(got, want), (shift, q, got)


def test_plain_results_replay_too():
    ids = np.array([2, 5, 9, 11, 400], np.uint32)
    off = np.array([0, 2, 2, 5], np.uint64)
    r = TrnResult()
    r.nq = 3
    r.offsets = off.ctypes.data_as(C.POINTER(C.c_uint64))
    r.docids = ids.ctypes.data_as(C.POINTER(C.c_uint32))
    for q, want in enumerate(([2, 5], [], [9, 11, 400])):
        rc, n, got = _decode(r, q, 8)
        assert rc == 0 and list(got) == want
    assert _decode(r, 3, 8)[0] == -1  # no such query


def test_malformed_segments_are_reported():
    r, keep = _compact([(0, [np.array([1, 2, 3], np.uint32)], [ENC_U16])], 12)
    keep[3][1] += 1  # the query claims one word more than its segments hold
    assert _decode(r, 0, 8)[0] == -3
    keep[3][1] -= 1
    # bucketed form whose count bytes do not add up to the item's documents
    r, keep = _compact([(0, [np.array([1, 2, 300, 301, 302], np.uint32)], [ENC_U8B])], 12)
    assert _decode(r, 0, 8)[0] == 0
    by = keep[0].view(np.uint8)
    by[1] += 1
    assert _decode(r, 0, 8)[0] == -3
    by[1] -= 2
    assert _decode(r, 0, 8)[0] == -3
