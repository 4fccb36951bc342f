// Flat plans (a conjunction or a disjunction whose operands are all terms — the ENT::matchallterms / ENT::matchanyterms runs of
// compilation_ctx.h:8-30, i.e. the 2-term AND and k-term OR workloads) in k_exec_docs.  (Included by exec_docs.cuh.)
//
// The per-tile blocks of ALL operand terms form one flat (term, block) list that the warp consumes 32 at a time, each lane decoding
// its block into the bitmap of ITS term; the conjunction is one word-wise AND at the end.  Compared with running the terms one after
// another this keeps the lanes full when a term has fewer than 32 blocks in the tile (the term-at-a-time path kept about a third
// of the lanes active per instruction).  When the rarest term is sparse inside the tile the caller falls back to the
// sequential path, whose advance()-style block skipping then saves more than the lane packing gains.
//
// Staging: every lane copies only the head of ITS block (kGatherBytes from the 16B-aligned address below the first doc-delta byte)
// with cp.async (LDGSTS) into its own slot — the doc-delta section of a 32-doc block is at most 31 x 2 bytes for gaps < 16384, and
// the inline hits behind it (half of the index bytes) never enter the SM.  (The span-copy version kept 6 KB per warp for one group,
// capped the SM at 20 resident warps and exposed every group's global-load latency.)
#pragma once

static constexpr uint32_t kFlatMaxLeaves = 16;

struct FlatLane { // per-lane description of one (term, block) work unit
        uint32_t j, off, n, prev, last;
        bool     active;
};

// returns 0 = not applicable (use the step program), 1 = handled (root docset in slot Q.root_slot), 2 = handled, result empty
__device__ int flat_exec_google(const ExecParams &P, const DevQuery &Q, uint32_t lo, uint32_t W, uint32_t NW, uint32_t *slots, uint8_t *stage, int lane) {
        const bool isAnd = Q.route == TRN_ROUTE_FLAT_AND;
        // lane j adopts the j-th leaf of the plan
        uint32_t nleaf = 0, myTerm = kEmptyTerm;
        for (uint32_t si = 0; si < Q.nsteps; ++si) {
                const DevStep st = P.steps[Q.step_begin + si];
                if (st.op == OP_LEAF) {
                        if (uint32_t(lane) == nleaf)
                                myTerm = st.term;
                        ++nleaf;
                }
        }
        if (nleaf == 0 || nleaf > kFlatMaxLeaves || (isAnd && nleaf > P.nslots))
                return 0;
        uint32_t mybA = 0, mycnt = 0, mydir = 0, mynb = 0, mydocs = 0, mydense = kDenseNone;
        if (uint32_t(lane) < nleaf && myTerm != kEmptyTerm) {
                const DevTerm T = P.ix.terms[myTerm];
                mydir           = T.dir_begin;
                mynb            = T.nblocks;
                mydocs          = T.documents;
                uint32_t a, b;
                tile_block_range(P.ix, T, lo, W, a, b);
                if (a <= b) {
                        mybA  = a;
                        mycnt = b - a + 1u;
                        // a conjunction's operand with a resident bitmap: the tile's words come from it (the tile lies inside the bitmap's span)
                        if (isAnd && P.ix.dense_off) {
                                const uint32_t o = __ldg(P.ix.dense_off + myTerm);
                                if (o != kDenseNone)
                                        mydense = o + ((lo - ((T.first_doc >> kDenseAlignShift) << kDenseAlignShift)) >> 5);
                        }
                }
        }
        unsigned dmask = 0; // conjunctions: the operands read from their bitmaps (not decoded)
        if (isAnd) {
                if (__ballot_sync(0xffffffffu, uint32_t(lane) < nleaf && mycnt == 0u))
                        return 2; // an operand has no posting in this tile
                dmask = __ballot_sync(0xffffffffu, mydense != kDenseNone);
                if (mydense != kDenseNone)
                        mycnt = 0;
        }
        const uint32_t incl  = warp_incl_scan(uint32_t(lane) < nleaf ? mycnt : 0u, lane);
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        if (isAnd) {
                // rarest decoded term (operands are sorted by df) sparse in this tile => skipping beats packing
                const unsigned dec = ~dmask & ((2u << (nleaf - 1u)) - 1u);
                if (dec) {
                        const uint32_t cnt0 = __shfl_sync(0xffffffffu, mycnt, __ffs(int(dec)) - 1);
                        if (64u * cnt0 < total - cnt0)
                                return 0;
                }
        } else if (total == 0u)
                return 2;

        uint32_t *     root   = slots + size_t(Q.root_slot) * NW;
        const uint32_t nclear = isAnd ? nleaf : 1u, lnw = P.exec_shift - 5u;
        for (uint32_t i = lane; i < nclear * NW; i += 32)
                if (!((dmask >> (i >> lnw)) & 1u)) // (the bitmap operands' slots are never read)
                        (isAnd ? slots : root)[i] = 0;

        // lane assignment of group g
        auto assign = [&](uint32_t g) {
                FlatLane       L;
                const uint32_t f = g + uint32_t(lane);
                L.active         = f < total;
                uint32_t j       = 0;
                for (uint32_t k = 0; k + 1u < nleaf; ++k)
                        j += (f >= __shfl_sync(0xffffffffu, incl, int(k))) ? 1u : 0u;
                if (!L.active)
                        j = nleaf - 1u;
                const uint32_t jincl = __shfl_sync(0xffffffffu, incl, int(j)), jcnt = __shfl_sync(0xffffffffu, mycnt, int(j));
                const uint32_t b     = __shfl_sync(0xffffffffu, mybA, int(j)) + (f - (jincl - jcnt));
                const uint32_t dir   = __shfl_sync(0xffffffffu, mydir, int(j));
                const uint32_t nb    = __shfl_sync(0xffffffffu, mynb, int(j));
                const uint32_t docs  = __shfl_sync(0xffffffffu, mydocs, int(j));
                L.j                  = j;
                L.off = L.n = L.prev = L.last = 0;
                if (L.active) {
                        const uint32_t *bl = P.ix.blk_last + dir, *bo = P.ix.blk_off + dir;
                        L.off  = bo[b];
                        L.last = bl[b];
                        L.prev = b ? bl[b - 1] : 0u;
                        L.n    = (b + 1u == nb) ? (docs - 32u * (nb - 1u)) : 32u;
                }
                return L;
        };

        // conjunctions: one bitmap per operand => plain-store word builder (OwnAcc); the last word of every block is ORed in
        // atomically one group LATER, after every block that can share it has stored its words
        const bool     own     = isAnd;
        const uint32_t dummy   = uint32_t(__cvta_generic_to_shared(stage + kGatherBufBytes)) + uint32_t(lane) * 4u;
        const uint32_t slots_s = uint32_t(__cvta_generic_to_shared(slots));
        uint32_t       tail_a = dummy, tail_bits = 0;
        FlatLane   cur  = assign(0);
        gather_issue(P.ix.index, cur.off, cur.active, stage, lane);
        __syncwarp(); // slot clears above are visible before the first reduction
        for (uint32_t g = 0; g < total; g += 32u) {
                const bool more = g + 32u < total;
                gather_wait<0>();
                const unsigned m = __ballot_sync(0xffffffffu, cur.active);
                if (own) {
                        OwnAcc bs;
                        bs.init(slots_s + cur.j * NW * 4u, dummy);
                        if (cur.active)
                                google_block_docs_vote(m, P.ix.index, cur.off, stage, lane, cur.n, cur.prev, cur.last, lo, W, bs);
                        __syncwarp();
                        if (tail_bits) // the previous group's last words
                                asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(tail_a), "r"(tail_bits) : "memory");
                        tail_a    = bs.cur_a;
                        tail_bits = bs.cur;
                } else if (cur.active) {
                        BitAcc bs;
                        bs.init(root);
                        google_block_docs_gather(m, P.ix.index, cur.off, stage, lane, cur.n, cur.prev, cur.last, lo, W, bs);
                        bs.flush();
                }
                __syncwarp();
                if (more) {
                        cur = assign(g + 32u);
                        gather_issue(P.ix.index, cur.off, cur.active, stage, lane);
                }
        }
        if (own && tail_bits)
                asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(tail_a), "r"(tail_bits) : "memory");
        __syncwarp();
        if (isAnd) {
                // operand i lives in slot i, or in its bitmap; the root of an all-term conjunction is slot 0
                const uint32_t NW4 = NW >> 2;
                const uint4 *  s4  = reinterpret_cast<const uint4 *>(slots);
                for (uint32_t i = lane; i < NW4; i += 32) {
                        uint4 w = make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu);
                        for (uint32_t k = 0; k < nleaf; ++k) {
                                const uint32_t dk = __shfl_sync(0xffffffffu, mydense, int(k));
                                const uint4    v  = dk != kDenseNone ? __ldg(reinterpret_cast<const uint4 *>(P.ix.dense + dk) + i) : s4[size_t(k) * NW4 + i];
                                w                 = make_uint4(w.x & v.x, w.y & v.y, w.z & v.z, w.w & v.w);
                        }
                        reinterpret_cast<uint4 *>(root)[i] = w;
                }
                __syncwarp();
        }
        return 1;
}

// One operand of a general step program decoded with the plain-store word builder: blocks [bA, bB] of term T into `out`, a bitmap
// that only this call writes (cleared by the caller).  Same loop as the conjunction case of flat_exec_google for a single term.
// `dummy`: shared address of 32 scratch words (one per lane).
__device__ void google_leaf_own(const DevIndex &ix, const DevTerm &T, uint32_t bA, uint32_t bB, uint32_t lo, uint32_t W, uint32_t *out, uint8_t *stage,
                                uint32_t dummy, int lane) {
        const uint32_t *bl = ix.blk_last + T.dir_begin, *bo = ix.blk_off + T.dir_begin;
        const uint32_t  out_s = uint32_t(__cvta_generic_to_shared(out));
        uint32_t        tail_a = dummy, tail_bits = 0;
        for (uint32_t g = bA; g <= bB; g += 32u) {
                const uint32_t b      = g + uint32_t(lane);
                const bool     active = b <= bB;
                uint32_t       off = 0, last = 0, prev = 0, n = 0;
                if (active) {
                        off  = bo[b];
                        last = bl[b];
                        prev = b ? bl[b - 1] : 0u;
                        n    = (b + 1u == T.nblocks) ? (T.documents - 32u * (T.nblocks - 1u)) : 32u;
                }
                gather_issue(ix.index, off, active, stage, lane);
                gather_wait<0>();
                const unsigned m = __ballot_sync(0xffffffffu, active);
                OwnAcc         bs;
                bs.init(out_s, dummy);
                if (active)
                        google_block_docs_vote(m, ix.index, off, stage, lane, n, prev, last, lo, W, bs);
                __syncwarp();
                if (tail_bits) // the previous group's last words, after every block that can share them has stored
                        asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(tail_a), "r"(tail_bits) : "memory");
                tail_a    = bs.cur_a;
                tail_bits = bs.cur;
        }
        if (tail_bits)
                asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(tail_a), "r"(tail_bits) : "memory");
        __syncwarp();
}

// ------------------------------------------------------------------------------------------------------------------------------------
// Flat-tree plans (DevQuery::route == TRN_ROUTE_FLAT_TREE): a DocumentsOnly tree that is neither an all-term run nor candidate-driven.  The host puts one
// [OP_LEAF M_NONE dst = j] marker per leaf at the front of the program (leaf j owns bitmap slot j) and turns the rest into slot operations.
// Per tile: ONE flat (leaf, block) pass decodes every leaf's blocks into its own bitmap with the plain-store word builder (lanes packed
// across leaves: the per-leaf groups of the step-program path ran at a third of the lanes), then the slot operations run as
// 128-bit vector operations.  Everything that depends only on the query — the leaves' term records, the slot operations (packed into one
// word each) — is loaded ONCE per query into lane registers (lane j: leaf j; lane k: operation k) and reused for all of its tiles.
struct TreeState {
        uint32_t dir, nb, docs, first, last, tfb, tfbase; // lane j < nleaf: leaf j
        uint32_t tfs;                                      // lane j < nleaf: leaf j's tf_shift
        uint32_t dense;                                    // lane j < nleaf: first word of leaf j's resident bitmap (kDenseNone: decoded)
        uint32_t op;                                       // lane k < nops: packed slot operation k
        uint32_t nleaf, nops;                              // (uniform)
};

__device__ __forceinline__ uint32_t tree_pack(const DevStep &st) {
        return uint32_t(st.op) | (uint32_t(st.mode) << 3) | (uint32_t(st.dst) << 6) | (uint32_t(st.src) << 11) | (uint32_t(st.flags & 3u) << 16) | ((st.term & 15u) << 18);
}

__device__ void tree_load(const ExecParams &P, const DevQuery &Q, TreeState &S, int lane) {
        S.nleaf = S.nops = 0;
        S.dir = S.nb = S.docs = S.first = S.last = S.tfb = S.tfbase = 0;
        S.tfs = 32;
        S.dense = kDenseNone;
        S.op = 0;
        uint32_t myTerm = kEmptyTerm;
        for (uint32_t si = 0; si < Q.nsteps; ++si) {
                const DevStep st = P.steps[Q.step_begin + si];
                if (st.op == OP_LEAF) { // markers: leaf S.nleaf owns slot S.nleaf
                        if (uint32_t(lane) == S.nleaf)
                                myTerm = st.term;
                        ++S.nleaf;
                } else {
                        if (uint32_t(lane) == S.nops)
                                S.op = tree_pack(st);
                        ++S.nops;
                }
        }
        if (uint32_t(lane) < S.nleaf && myTerm != kEmptyTerm) {
                const DevTerm T = P.ix.terms[myTerm];
                S.dir    = T.dir_begin;
                S.nb     = T.nblocks;
                S.docs   = T.documents;
                S.first  = T.first_doc;
                S.last   = T.last_doc;
                S.tfb    = T.tf_begin;
                S.tfbase = T.tf_base;
                S.tfs    = T.tf_shift;
                if (P.ix.dense_off)
                        S.dense = __ldg(P.ix.dense_off + myTerm);
        }
}

// returns true when the plan's F_BREAK_IF_EMPTY fired (the tile matches nothing); else the root docset is in slot Q.root_slot.
__device__ bool tree_exec_google(const ExecParams &P, const DevQuery &Q, const TreeState &S, uint32_t lo, uint32_t W, uint32_t NW, uint32_t *slots, uint8_t *stage, int lane) {
        const uint32_t nleaf = S.nleaf;
        // ---- leaf bitmaps start empty
        {
                uint4 *        s4 = reinterpret_cast<uint4 *>(slots);
                const uint32_t n4 = nleaf * (NW >> 2);
                for (uint32_t i = lane; i < n4; i += 32)
                        s4[i] = make_uint4(0, 0, 0, 0);
        }
        const uint32_t dummy   = uint32_t(__cvta_generic_to_shared(stage + kGatherBufBytes)) + uint32_t(lane) * 4u;
        const uint32_t slots_s = uint32_t(__cvta_generic_to_shared(slots));
        const uint32_t NW4     = NW >> 2;
        const uint32_t past    = P.ix.max_docid < 0x80000000u ? 0x80000000u - W : 0u;
        __syncwarp(); // the clears above are visible before the first store
        // ---- leaves with a resident bitmap: a vector copy of the tile's words (the tile lies inside the bitmap's span)
        const bool inTile = uint32_t(lane) < nleaf && S.nb && lo <= S.last && lo + (W - 1u) >= S.first;
        for (unsigned dm = __ballot_sync(0xffffffffu, inTile && S.dense != kDenseNone); dm; dm &= dm - 1u) {
                const int      j  = __ffs(int(dm)) - 1;
                const uint32_t f  = __shfl_sync(0xffffffffu, S.first, j);
                const uint4 *  s4 = reinterpret_cast<const uint4 *>(P.ix.dense + __shfl_sync(0xffffffffu, S.dense, j) +
                                                                   ((lo - ((f >> kDenseAlignShift) << kDenseAlignShift)) >> 5));
                uint4 *d4 = reinterpret_cast<uint4 *>(slots) + size_t(j) * NW4;
                for (uint32_t i = lane; i < NW4; i += 32)
                        d4[i] = __ldg(s4 + i);
        }
        // ---- the tile's blocks of every other leaf
        uint32_t mybA = 0, mycnt = 0;
        if (inTile && S.dense == kDenseNone) {
                const uint32_t a = first_block_ge(P.ix, S.dir, S.nb, S.first, S.last, S.tfb, S.tfbase, S.tfs, lo);
                if (a < S.nb) {
                        const uint32_t hi = lo + W; // wraps to 0 for the last tile of a 2^32 docID space
                        const uint32_t e  = (hi == 0u || hi > S.last) ? S.nb : first_block_ge(P.ix, S.dir, S.nb, S.first, S.last, S.tfb, S.tfbase, S.tfs, hi);
                        mybA              = a;
                        mycnt             = min(e, S.nb - 1u) - a + 1u;
                }
        }
        const uint32_t incl  = warp_incl_scan(mycnt, lane);
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        // lane assignment of the group that starts at flat entry g; all lanes take part
        auto assign = [&](uint32_t g) {
                FlatLane       L;
                const uint32_t f = g + uint32_t(lane);
                L.active         = f < total;
                uint32_t j       = 0;
                for (uint32_t k = 0; k + 1u < nleaf; ++k)
                        j += (f >= __shfl_sync(0xffffffffu, incl, int(k))) ? 1u : 0u;
                if (!L.active)
                        j = nleaf - 1u;
                const uint32_t jincl = __shfl_sync(0xffffffffu, incl, int(j)), jcnt = __shfl_sync(0xffffffffu, mycnt, int(j));
                const uint32_t b     = __shfl_sync(0xffffffffu, mybA, int(j)) + (f - (jincl - jcnt));
                const uint32_t dir   = __shfl_sync(0xffffffffu, S.dir, int(j));
                const uint32_t nb    = __shfl_sync(0xffffffffu, S.nb, int(j));
                const uint32_t docs  = __shfl_sync(0xffffffffu, S.docs, int(j));
                L.j                  = j;
                L.off = L.n = L.prev = L.last = 0;
                if (L.active) {
                        const uint32_t *bl = P.ix.blk_last + dir, *bo = P.ix.blk_off + dir;
                        L.off  = __ldg(bo + b);
                        L.last = __ldg(bl + b);
                        L.prev = b ? __ldg(bl + b - 1u) : 0u;
                        L.n    = (b + 1u == nb) ? (docs - 32u * (nb - 1u)) : 32u;
                }
                return L;
        };
        uint32_t tail_a = dummy, tail_bits = 0;
        FlatLane cur;
        if (total) {
                cur = assign(0);
                gather_issue(P.ix.index, cur.off, cur.active, stage, lane);
        }
        for (uint32_t g = 0; g < total; g += 32u) {
                gather_wait<0>();
                OwnAcc bs;
                bs.init(slots_s + cur.j * NW * 4u, dummy);
                if (cur.active)
                        google_block_docs_lane(P.ix.index, cur.off, stage, lane, cur.n, cur.prev, cur.last, lo, W, bs, past);
                __syncwarp();
                if (tail_bits) // the previous group's last words, after every block that can share them has stored
                        asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(tail_a), "r"(tail_bits) : "memory");
                tail_a    = bs.cur_a;
                tail_bits = bs.cur;
                if (g + 32u < total) {
                        cur = assign(g + 32u);
                        gather_issue(P.ix.index, cur.off, cur.active, stage, lane);
                }
        }
        if (tail_bits)
                asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(tail_a), "r"(tail_bits) : "memory");
        __syncwarp();
        // ---- slot operations, 128 bits per lane and step
        for (uint32_t k = 0; k < S.nops; ++k) {
                const uint32_t w    = __shfl_sync(0xffffffffu, S.op, int(k));
                const uint32_t op   = w & 7u, mode = (w >> 3) & 7u, dsti = (w >> 6) & 31u, srci = (w >> 11) & 31u, flags = (w >> 16) & 3u, arg = (w >> 18) & 15u;
                uint4 *        d4   = reinterpret_cast<uint4 *>(slots + size_t(dsti) * NW);
                const uint4 *  s4   = reinterpret_cast<const uint4 *>(slots + size_t(srci) * NW);
                if (op == OP_CLEAR) {
                        for (uint32_t i = lane; i < NW4; i += 32)
                                d4[i] = make_uint4(0, 0, 0, 0);
                } else if (op == OP_SLOT) {
                        if (mode == M_SET) {
                                for (uint32_t i = lane; i < NW4; i += 32)
                                        d4[i] = s4[i];
                        } else if (mode == M_OR) {
                                for (uint32_t i = lane; i < NW4; i += 32) {
                                        const uint4 a = d4[i], b = s4[i];
                                        d4[i]         = make_uint4(a.x | b.x, a.y | b.y, a.z | b.z, a.w | b.w);
                                }
                        } else if (mode == M_AND) {
                                for (uint32_t i = lane; i < NW4; i += 32) {
                                        const uint4 a = d4[i], b = s4[i];
                                        d4[i]         = make_uint4(a.x & b.x, a.y & b.y, a.z & b.z, a.w & b.w);
                                }
                        } else if (mode == M_ANDNOT) {
                                for (uint32_t i = lane; i < NW4; i += 32) {
                                        const uint4 a = d4[i], b = s4[i];
                                        d4[i]         = make_uint4(a.x & ~b.x, a.y & ~b.y, a.z & ~b.z, a.w & ~b.w);
                                }
                        }
                } else if (op == OP_COUNT_ADD) { // bit-sliced saturating counters (DisjunctionSome): plane j lives in slot dst + j, `mode` planes
                        const uint32_t *src = slots + size_t(srci) * NW;
                        for (uint32_t i = lane; i < NW; i += 32) {
                                uint32_t carry = src[i];
                                for (uint32_t j = 0; j < mode && carry; ++j) {
                                        uint32_t *     pl = slots + size_t(dsti + j) * NW;
                                        const uint32_t p  = pl[i];
                                        pl[i]             = p ^ carry;
                                        carry &= p;
                                }
                                if (carry)
                                        for (uint32_t j = 0; j < mode; ++j)
                                                slots[size_t(dsti + j) * NW + i] |= carry;
                        }
                } else if (op == OP_COUNT_GE) {
                        uint32_t *dst = slots + size_t(dsti) * NW;
                        for (uint32_t i = lane; i < NW; i += 32) {
                                uint32_t gt = 0, eq = 0xffffffffu;
                                for (int j = int(mode) - 1; j >= 0; --j) {
                                        const uint32_t p = slots[size_t(srci + j) * NW + i];
                                        if ((arg >> j) & 1u) eq &= p;
                                        else gt |= eq & p;
                                }
                                dst[i] = gt | eq;
                        }
                }
                __syncwarp();
                if (flags & F_BREAK_IF_EMPTY) {
                        uint32_t any = 0;
                        for (uint32_t i = lane; i < NW4; i += 32) {
                                const uint4 a = d4[i];
                                any |= a.x | a.y | a.z | a.w;
                        }
                        if (!__any_sync(0xffffffffu, any != 0u))
                                return true;
                }
        }
        return false;
}
