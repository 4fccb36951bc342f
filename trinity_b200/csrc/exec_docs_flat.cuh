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
        uint32_t mybA = 0, mycnt = 0, mydir = 0, mynb = 0, mydocs = 0;
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
                }
        }
        const uint32_t incl  = warp_incl_scan(uint32_t(lane) < nleaf ? mycnt : 0u, lane);
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        if (isAnd) {
                if (__ballot_sync(0xffffffffu, uint32_t(lane) < nleaf && mycnt == 0u))
                        return 2; // an operand has no posting in this tile
                // rarest term (operands are sorted by df) sparse in this tile => skipping beats packing
                const uint32_t cnt0 = __shfl_sync(0xffffffffu, mycnt, 0);
                if (64u * cnt0 < total - cnt0)
                        return 0;
        } else if (total == 0u)
                return 2;

        uint32_t *     root   = slots + size_t(Q.root_slot) * NW;
        const uint32_t nclear = isAnd ? nleaf : 1u;
        for (uint32_t i = lane; i < nclear * NW; i += 32)
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
                // operand i lives in slot i; the root of an all-term conjunction is slot 0
                for (uint32_t i = lane; i < NW; i += 32) {
                        uint32_t w = slots[i];
                        for (uint32_t k = 1; k < nleaf; ++k)
                                w &= slots[size_t(k) * NW + i];
                        root[i] = w;
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
        uint32_t tfs;                                      // bits 0-7: tf_shift; 8-12: mask slot; 16: decoded in the masked second pass
        uint32_t op, mop;                                  // lane k < nops / nmops: packed slot operation k of the main / mask section
        uint32_t nleaf, nops, nmops, nmasked;              // (uniform)
};

__device__ __forceinline__ uint32_t tree_pack(const DevStep &st) {
        return uint32_t(st.op) | (uint32_t(st.mode) << 3) | (uint32_t(st.dst) << 6) | (uint32_t(st.src) << 11) | (uint32_t(st.flags & 3u) << 16) | ((st.term & 15u) << 18);
}

__device__ void tree_load(const ExecParams &P, const DevQuery &Q, TreeState &S, int lane) {
        S.nleaf = S.nops = S.nmops = S.nmasked = 0;
        S.dir = S.nb = S.docs = S.first = S.last = S.tfb = S.tfbase = 0;
        S.tfs = 32;
        S.op = S.mop = 0;
        uint32_t myTerm = kEmptyTerm, myMask = 0;
        for (uint32_t si = 0; si < Q.nsteps; ++si) {
                const DevStep st = P.steps[Q.step_begin + si];
                if (st.op == OP_LEAF) { // markers: leaf S.nleaf owns slot S.nleaf
                        if (uint32_t(lane) == S.nleaf) {
                                myTerm = st.term;
                                myMask = (st.flags & F_MASKED) ? (0x10000u | (uint32_t(st.src) << 8)) : 0u;
                        }
                        S.nmasked += (st.flags & F_MASKED) ? 1u : 0u;
                        ++S.nleaf;
                } else if (st.flags & F_MASKOP) {
                        if (uint32_t(lane) == S.nmops)
                                S.mop = tree_pack(st);
                        ++S.nmops;
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
        }
        S.tfs |= myMask;
}

// returns true when the plan's F_BREAK_IF_EMPTY fired (the tile matches nothing); else the root docset is in slot Q.root_slot.
// Two decode passes (planner.cpp: flat_tree_masks): pass 0 decodes the first-pass leaves and runs the mask section; pass 1 decodes, of the
// masked leaves, only the blocks whose docID range holds a set bit of their mask bitmap, and runs the plan's own slot operations.
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
        uint32_t *     queue   = reinterpret_cast<uint32_t *>(stage + kGatherBufBytes + 128u); // 64 entries: the needed (leaf, block) pairs of pass 1
        const uint32_t NW4     = NW >> 2;
        const uint32_t past    = P.ix.max_docid < 0x80000000u ? 0x80000000u - W : 0u;
        __syncwarp(); // the clears above are visible before the first store
        for (uint32_t pass = 0; pass < 2u; ++pass) {
                const bool masked = pass != 0u;
                if (!masked || S.nmasked) {
                        // ---- the tile's blocks of every leaf of this pass
                        uint32_t mybA = 0, mycnt = 0;
                        if (uint32_t(lane) < nleaf && S.nb && ((S.tfs >> 16) & 1u) == pass && lo <= S.last && lo + (W - 1u) >= S.first) {
                                const uint32_t tfs = S.tfs & 0xffu;
                                const uint32_t a   = first_block_ge(P.ix, S.dir, S.nb, S.first, S.last, S.tfb, S.tfbase, tfs, lo);
                                if (a < S.nb) {
                                        const uint32_t hi = lo + W; // wraps to 0 for the last tile of a 2^32 docID space
                                        const uint32_t e  = (hi == 0u || hi > S.last) ? S.nb : first_block_ge(P.ix, S.dir, S.nb, S.first, S.last, S.tfb, S.tfbase, tfs, hi);
                                        mybA              = a;
                                        mycnt             = min(e, S.nb - 1u) - a + 1u;
                                }
                        }
                        const uint32_t incl  = warp_incl_scan(mycnt, lane);
                        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
                        // (leaf, block) of flat entry f; all lanes take part
                        auto locate = [&](uint32_t f, bool act, uint32_t &j, uint32_t &b) {
                                j = 0;
                                for (uint32_t k = 0; k + 1u < nleaf; ++k)
                                        j += (f >= __shfl_sync(0xffffffffu, incl, int(k))) ? 1u : 0u;
                                if (!act)
                                        j = nleaf - 1u;
                                const uint32_t jincl = __shfl_sync(0xffffffffu, incl, int(j)), jcnt = __shfl_sync(0xffffffffu, mycnt, int(j));
                                b                    = __shfl_sync(0xffffffffu, mybA, int(j)) + (f - (jincl - jcnt));
                        };
                        auto fill = [&](FlatLane &L, uint32_t j, uint32_t b) {
                                const uint32_t dir  = __shfl_sync(0xffffffffu, S.dir, int(j));
                                const uint32_t nb   = __shfl_sync(0xffffffffu, S.nb, int(j));
                                const uint32_t docs = __shfl_sync(0xffffffffu, S.docs, int(j));
                                L.j                 = j;
                                L.off = L.n = L.prev = L.last = 0;
                                if (L.active) {
                                        const uint32_t *bl = P.ix.blk_last + dir, *bo = P.ix.blk_off + dir;
                                        L.off  = __ldg(bo + b);
                                        L.last = __ldg(bl + b);
                                        L.prev = b ? __ldg(bl + b - 1u) : 0u;
                                        L.n    = (b + 1u == nb) ? (docs - 32u * (nb - 1u)) : 32u;
                                }
                        };
                        uint32_t fnext = 0, qhead = 0, qn = 0; // (uniform) next unexamined flat entry; the queue of pass 1
                        // the next group of up to 32 blocks to decode; returns false when the pass is done
                        auto next = [&](FlatLane &L) -> bool {
                                if (!masked) {
                                        if (fnext >= total)
                                                return false;
                                        const uint32_t f = fnext + uint32_t(lane);
                                        fnext += 32u;
                                        L.active = f < total;
                                        uint32_t j, b;
                                        locate(f, L.active, j, b);
                                        fill(L, j, b);
                                        return true;
                                }
                                while (qn < 32u && fnext < total) { // examine 32 more entries: does the mask hold a docID of the block's range?
                                        const uint32_t f   = fnext + uint32_t(lane);
                                        const bool     act = f < total;
                                        fnext += 32u;
                                        uint32_t j, b;
                                        locate(f, act, j, b);
                                        const uint32_t dir = __shfl_sync(0xffffffffu, S.dir, int(j));
                                        const uint32_t ms  = (__shfl_sync(0xffffffffu, S.tfs, int(j)) >> 8) & 31u;
                                        bool           need{false};
                                        if (act) {
                                                const uint32_t *bl   = P.ix.blk_last + dir;
                                                const uint32_t  last = __ldg(bl + b), prev = b ? __ldg(bl + b - 1u) : 0u;
                                                const uint32_t  d0 = max(prev + 1u, lo), d1 = min(last, lo + (W - 1u));
                                                if (d0 <= d1) {
                                                        const uint32_t  r0 = d0 - lo, r1 = d1 - lo;
                                                        const uint32_t *M  = slots + size_t(ms) * NW;
                                                        uint32_t        w = r0 >> 5, v = M[w] & (0xffffffffu << (r0 & 31u));
                                                        const uint32_t  w1 = r1 >> 5;
                                                        while (w < w1 && !v)
                                                                v = M[++w];
                                                        if (w == w1)
                                                                v &= 0xffffffffu >> (31u - (r1 & 31u));
                                                        need = v != 0u;
                                                }
                                        }
                                        const unsigned m = __ballot_sync(0xffffffffu, need);
                                        if (need)
                                                queue[(qhead + qn + __popc(m & ((1u << lane) - 1u))) & 63u] = (j << 28) | b;
                                        qn += __popc(m);
                                }
                                if (!qn)
                                        return false;
                                __syncwarp();
                                const uint32_t take = min(qn, 32u);
                                L.active            = uint32_t(lane) < take;
                                const uint32_t e    = L.active ? queue[(qhead + uint32_t(lane)) & 63u] : 0u;
                                qhead += take;
                                qn -= take;
                                fill(L, e >> 28, e & 0x0fffffffu);
                                return true;
                        };
                        uint32_t tail_a = dummy, tail_bits = 0;
                        FlatLane cur;
                        bool     more = next(cur);
                        if (more)
                                gather_issue(P.ix.index, cur.off, cur.active, stage, lane);
                        while (more) {
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
                                more      = next(cur);
                                if (more)
                                        gather_issue(P.ix.index, cur.off, cur.active, stage, lane);
                        }
                        if (tail_bits)
                                asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(tail_a), "r"(tail_bits) : "memory");
                        __syncwarp();
                }
                // ---- slot operations of this pass (pass 0: the mask section), 128 bits per lane and step
                const uint32_t cnt = masked ? S.nops : S.nmops;
                const uint32_t reg = masked ? S.op : S.mop;
                for (uint32_t k = 0; k < cnt; ++k) {
                        const uint32_t w    = __shfl_sync(0xffffffffu, reg, int(k));
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
        }
        return false;
}
