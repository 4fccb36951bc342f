"""CPU interpreter of the bitmap-path step programs the plan compiler emits (trn_debug_compile): the same slot algebra the exec kernels
run per docID tile, over whole-index boolean arrays.  TEST INFRASTRUCTURE: lets plan-compiler changes be checked without a GPU."""
import numpy as np

import trinity_b200 as tb

OP_LEAF, OP_SLOT, OP_CLEAR, OP_LEAFSCORE, OP_COUNT_ADD, OP_COUNT_GE = 0, 1, 2, 3, 4, 5
M_SET, M_OR, M_AND, M_ANDNOT, M_NONE = 0, 1, 2, 3, 4
F_SCORE, F_BREAK_IF_EMPTY = 1, 2


def run(steps, root_slot, nslots, lists, ndocs, tree=False):
    """returns (match[ndocs+1], score[ndocs+1]); lists[t] = (docids, freqs).  tree: a flat-tree program — its leading
    [LEAF, mode NONE, dst] markers name bitmaps that one flat decode pass fills before the slot operations run"""
    slots = [np.zeros(ndocs + 1, bool) for _ in range(nslots)]
    acc = np.zeros(ndocs + 1, np.float32)  # the kernels accumulate fp32 scores in step order
    dead = False

    def leaf(term):
        m = np.zeros(ndocs + 1, bool)
        s = None
        if term != tb.EMPTY_TERM:
            d, f = lists[term]
            m[d] = True
            s = (d, f)
        return m, s

    for st in steps:
        if dead:
            break
        op, mode, dst, src = int(st["op"]), int(st["mode"]), int(st["dst"]), int(st["src"])
        if op == OP_CLEAR:
            slots[dst][:] = False
        elif op == OP_SLOT:
            if mode == M_SET: slots[dst] = slots[src].copy()
            elif mode == M_OR: slots[dst] |= slots[src]
            elif mode == M_AND: slots[dst] &= slots[src]
            elif mode == M_ANDNOT: slots[dst] &= ~slots[src]
        elif op in (OP_LEAF, OP_LEAFSCORE):
            m, s = leaf(int(st["term"]))
            if op == OP_LEAF:
                if tree and mode == M_NONE:
                    slots[dst] = m.copy()
                if mode == M_SET: slots[dst] = m.copy()
                elif mode == M_OR: slots[dst] |= m
                elif mode == M_AND: slots[dst] &= m
                elif mode == M_ANDNOT: slots[dst] &= ~m
                if (int(st["flags"]) & F_SCORE) and s is not None:
                    d, f = s
                    acc[d] += np.array([tb.bm25_score(float(st["idf"]), int(x) & 0xFFFF) for x in f], np.float32)
            elif s is not None:
                d, f = s
                keep = slots[src][d]
                acc[d[keep]] += np.array([tb.bm25_score(float(st["idf"]), int(x) & 0xFFFF) for x in f[keep]], np.float32)
        elif op == OP_COUNT_ADD:
            carry = slots[src].copy()
            for j in range(mode):
                p = slots[dst + j]
                slots[dst + j] = p ^ carry
                carry = p & carry
            for j in range(mode):  # saturate
                slots[dst + j] |= carry
        elif op == OP_COUNT_GE:
            m = int(st["term"])
            gt = np.zeros(ndocs + 1, bool)
            eq = np.ones(ndocs + 1, bool)
            for j in range(mode - 1, -1, -1):
                p = slots[src + j]
                if (m >> j) & 1: eq &= p
                else: gt |= eq & p
            slots[dst] = gt | eq
        else:
            raise AssertionError(f"unknown step op {op}")
        if op in (OP_LEAF, OP_SLOT) and (int(st["flags"]) & F_BREAK_IF_EMPTY) and not slots[dst].any():
            dead = True
    if dead:
        return np.zeros(ndocs + 1, bool), np.zeros(ndocs + 1, np.float64)
    match = slots[root_slot].copy()
    match[0] = False
    return match, np.where(match, acc.astype(np.float64), 0.0)
