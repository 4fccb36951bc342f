// k_exec_docs — DocumentsOnly execution with one WARP per work item.  (Included by kernels.cu.)
//
// A work item is a (query, docID tile) pair for the bitmap paths (general step programs here, all-term conjunctions / disjunctions in
// exec_docs_flat.cuh) or a 32-block group of a lead term for the candidate-driven path (exec_docs_cand.cuh); the host picks the path
// per query (planner.cpp, plan_batch: DevQuery::route).
//
// Why a second kernel: the ncu capture of the CTA-per-tile kernel on the 2-term AND workload showed DRAM far from
// peak, low issue utilisation and half of all stall samples on CTA barriers — 4 warps waiting for the slowest lane-serial block
// decode at every step.  Set queries need no score tile, so the whole per-tile state (2-3 slot bitmaps + one staging area) fits a
// warp: every warp is an independent worker that never waits for another warp (only __syncwarp), and the SM always has
// as many runnable decode chains as it has resident warps.
//
// Same step programs, same decode routines, same output contract as k_exec_tiles (mode TRN_MODE_DOCS_ONLY).
#pragma once

static constexpr int      kDocsWarps       = 4;   // warps per CTA (independent workers)
static constexpr uint32_t kSparseThreshold = 192; // candidates per tile below which AND switches to advance()-style skipping
static constexpr uint32_t kGatherBytes     = 80;  // bytes of a block's head each lane stages (5 x 16 B; >= 64 payload bytes after alignment)
static constexpr uint32_t kGatherBufBytes  = 32 * kGatherBytes;  // one group
// per-warp staging: ONE gather buffer + a 128-word area (need-list of the block-skipping path / scratch words of the word builders / Lucene
// exception patches).  A second, prefetching buffer was measured and dropped: it costs a quarter of the resident warps (24 instead of 32
// per SM) and made the headline batch slower.
static constexpr uint32_t kDocsStageBytes1 = kGatherBufBytes + 512;

// ---- lane-gather staging with cp.async (LDGSTS): no registers, no L1 allocation, completion tracked per group
__device__ __forceinline__ void gather_issue(const uint8_t *__restrict__ index, uint32_t off, bool need, uint8_t *buf, int lane) {
        if (need) {
                const uint8_t *src = index + (off & ~15u);
                const uint32_t dst = uint32_t(__cvta_generic_to_shared(buf + lane * kGatherBytes));
#pragma unroll
                for (uint32_t c = 0; c < kGatherBytes; c += 16u)
                        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + c), "l"(src + c) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N> __device__ __forceinline__ void gather_wait() {
        asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
        __syncwarp();
}

// lower_bound over bl[a..b] (ascending) for the first index with bl[idx] >= v; returns b+1 if none.  Warp-cooperative 32-ary search.
__device__ __forceinline__ uint32_t warp_lower_bound(const uint32_t *__restrict__ bl, uint32_t a, uint32_t b, uint32_t v, int lane) {
        // invariant: answer in [a, b+1]
        while (b - a + 1u > 32u) {
                const uint32_t n = b - a + 1u, step = (n + 31u) / 32u;
                const uint32_t p = min(b, a + uint32_t(lane) * step + (step - 1u)); // last element of chunk `lane`
                const uint32_t c = __popc(__ballot_sync(0xffffffffu, bl[p] < v)); // chunks entirely < v (monotone)
                if (c == 32u)
                        return b + 1u;
                const uint32_t na = a + c * step;
                b                 = min(b, na + step - 1u);
                a                 = na;
        }
        const uint32_t idx = a + uint32_t(lane);
        const uint32_t val = idx <= b ? bl[idx] : 0xffffffffu;
        return a + __popc(__ballot_sync(0xffffffffu, val < v));
}

// docs-only visitor: word-register bit builder (see BitSink)
struct DocSink {
        BitSink bits;
        __device__ __forceinline__ void visit(uint32_t rel) {
                bits.add(rel);
        }
};

// lean word-register bit builder (or-in only, no filter): one shared-memory reduction per touched 32-doc word.
// The flush is a single PREDICATED red.shared.or (no branch): with a branch, the two or three lanes of a warp that cross a word
// boundary at any given posting made the whole warp execute the flush body at ~2/32 lane occupancy on almost every posting.
struct BitAcc {
        uint32_t bm;    // shared-state-space address of the bitmap
        uint32_t cur_w, cur;
        __device__ __forceinline__ void init(uint32_t *b) {
                bm    = uint32_t(__cvta_generic_to_shared(b));
                cur_w = 0;
                cur   = 0;
        }
        __device__ __forceinline__ void red_if(uint32_t flag) {
                asm volatile("{ .reg .pred p; setp.ne.u32 p, %2, 0; @p red.shared.or.b32 [%0], %1; }" ::"r"(bm + cur_w * 4u), "r"(cur), "r"(flag) : "memory");
        }
        __device__ __forceinline__ void add(uint32_t rel) {
                const uint32_t w = rel >> 5, bit = 1u << (rel & 31u);
                const bool     nw = w != cur_w;
                red_if((nw && cur) ? 1u : 0u);
                cur   = nw ? bit : (cur | bit);
                cur_w = w;
        }
        __device__ __forceinline__ void flush() {
                red_if(cur);
                cur = 0;
        }
};

__device__ __forceinline__ uint32_t lds_u8(uint32_t saddr) {
        uint32_t v;
        asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(saddr));
        return v;
}

// Byte-wise decoder over the lane's gather slot.  The span-staged whole-list decoder (plain byte loads) needs about
// two warp-instructions per posting for deltas AND freqs with nearly all lanes active, fewer than the 64-bit-window decoder
// spends on deltas alone: a 1-byte code costs one LDS.U8, one compare and the adds.  Codes of up to two bytes (gaps < 16384) always
// lie inside the 80-byte slot (31 x 2 + 15 bytes of alignment slack); the first longer code switches the lane to global memory.
template <class SINK>
__device__ __forceinline__ void google_block_docs_bytes(const uint8_t *__restrict__ index, uint32_t off, const uint8_t *buf, int lane, uint32_t n, uint32_t prev,
                                                        uint32_t last, uint32_t lo, uint32_t W, SINK &bs) {
        const uint32_t mis = off & 15u;
        uint32_t       sp  = uint32_t(__cvta_generic_to_shared(buf + lane * kGatherBytes)) + mis; // shared address of the first delta byte
        const uint32_t nd  = n - 1u;
        uint32_t       doc = prev, i = 0, p = 0;
        for (; i < nd; ++i) {
                const uint32_t b0 = lds_u8(sp + p);
                uint32_t       v;
                if (b0 < 0x80u) {
                        v = b0;
                        p += 1u;
                } else if (b0 < 0xc0u) {
                        v = ((b0 & 0x3fu) << 8) | lds_u8(sp + p + 1u);
                        p += 2u;
                } else
                        break; // 3..5-byte code: the section may leave the slot
                doc += v;
                if (doc - lo < W)
                        bs.add(doc - lo);
        }
        if (i < nd) {
                const uint8_t *g = index + off + p;
                for (; i < nd; ++i) {
                        doc += varbyte_get(g);
                        if (doc - lo < W)
                                bs.add(doc - lo);
                }
        }
        if (last - lo < W)
                bs.add(last - lo);
}

__device__ __forceinline__ uint32_t lds_u32(uint32_t saddr) {
        uint32_t v;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr));
        return v;
}

// Plain-store word builder for a bitmap that only ONE term writes (flat conjunctions keep one slot per operand).  The blocks of
// a term partition the docID space, so every 32-doc word strictly between a block's first and last word belongs to that block's
// lane alone: it is written with a predicated STS when the lane moves on — no atomic, and no branch (ptxas turns a predicated
// red.shared into BSSY / BRA / ATOMS / BSYNC: three control instructions per posting and branch-resolve stalls).  Only a block's LAST word can be shared, with the following block(s) of the term; the caller ORs it in
// atomically AFTER those have stored (see flat_exec_google).
struct OwnAcc {
        uint32_t bm;           // shared-state-space address of the term's bitmap
        uint32_t cur_w, cur_a; // word being accumulated, and where it goes when the lane leaves it
        uint32_t cur;
        __device__ __forceinline__ void init(uint32_t bm_saddr, uint32_t dummy_saddr) {
                bm    = bm_saddr;
                asm volatile("" : "+r"(bm)); // keep the base in a register (one LEA per posting instead of recomputing slot * NW)
                cur_w = 0xffffffffu;
                cur_a = dummy_saddr; // the first "flush" stores an empty accumulator here
                cur   = 0;
        }
        __device__ __forceinline__ void add(uint32_t rel) {
                const uint32_t w = rel >> 5, bit = __funnelshift_l(0u, 1u, rel); // 1 << (rel & 31)
                const uint32_t nw = w != cur_w ? 1u : 0u;
                asm volatile("{ .reg .pred p; setp.ne.u32 p, %2, 0; @p st.shared.u32 [%0], %1; }" ::"r"(cur_a), "r"(cur), "r"(nw) : "memory");
                cur   = (nw ? 0u : cur) | bit;
                cur_w = w;
                cur_a = bm + w * 4u;
        }
};

// OwnAcc::add under a per-lane predicate, branch-free (every lane of the warp executes the same instructions)
__device__ __forceinline__ void own_add_if(OwnAcc &bs, bool on, uint32_t rel) {
        const uint32_t w = rel >> 5, bit = __funnelshift_l(0u, 1u, rel);
        const uint32_t nw = (on && w != bs.cur_w) ? 1u : 0u;
        asm volatile("{ .reg .pred p; setp.ne.u32 p, %2, 0; @p st.shared.u32 [%0], %1; }" ::"r"(bs.cur_a), "r"(bs.cur), "r"(nw) : "memory");
        bs.cur   = (nw ? 0u : bs.cur) | (on ? bit : 0u);
        bs.cur_w = on ? w : bs.cur_w;
        bs.cur_a = on ? bs.bm + w * 4u : bs.cur_a;
}

// Warp-voted decoder into an OwnAcc.  Its predecessor let every lane choose between a 4-wide body and byte-wise excursions on its
// own, which cost this: few of the 4-byte words hold a 2-byte code, but each of them sent its
// warp through ~3 byte-wise iterations at a few of 32 lanes — more instructions than the 4-wide body itself.  Here every iteration reads a 32-bit window at ANY byte position (two aligned shared loads + funnel shift:
// no alignment prologue, no re-alignment), and the warp votes: all lanes see four 1-byte codes => the 4-wide body; otherwise ALL
// lanes run one predicated, branch-free step that consumes the leading 1-byte codes of the window plus the first 2-byte code
// (1..4 postings).  The two bodies are never executed in the same iteration.
__device__ __forceinline__ void google_block_docs_vote(unsigned m, const uint8_t *__restrict__ index, uint32_t off, const uint8_t *buf, int lane, uint32_t n,
                                                       uint32_t prev, uint32_t last, uint32_t lo, uint32_t W, OwnAcc &bs) {
        const uint32_t mis  = off & 15u;
        const uint32_t base = uint32_t(__cvta_generic_to_shared(buf + lane * kGatherBytes)) + mis; // shared address of the first delta byte
        const uint32_t nd   = n - 1u;
        uint32_t       sp = base, rel = prev - lo, i = 0;
        bool           spill = false; // met a 3..5-byte code: the section may leave the slot
        for (;;) {
                const bool live = i < nd && !spill;
                if (!__any_sync(m, live))
                        break;
                const uint32_t a  = sp & ~3u;
                const uint32_t w  = __funnelshift_r(lds_u32(a), lds_u32(a + 4u), (sp & 3u) * 8u); // bytes sp .. sp+3
                const uint32_t hb = w & 0x80808080u, rem = nd - i;
                const uint32_t b0 = w & 0xffu, b1 = __byte_perm(w, 0u, 0x4441u), b2 = __byte_perm(w, 0u, 0x4442u), b3 = w >> 24;
                if (__all_sync(m, !live || (hb == 0u && rem >= 4u))) {
                        if (live) {
                                const uint32_t r0 = rel + b0, r1 = r0 + b1, r2 = r1 + b2, r3 = r2 + b3;
                                rel = r3;
                                sp += 4u;
                                i += 4u;
                                if (r0 < W && r3 < W) {
                                        bs.add(r0);
                                        bs.add(r1);
                                        bs.add(r2);
                                        bs.add(r3);
                                } else {
                                        own_add_if(bs, r0 < W, r0);
                                        own_add_if(bs, r1 < W, r1);
                                        own_add_if(bs, r2 < W, r2);
                                        own_add_if(bs, r3 < W, r3);
                                }
                        }
                } else {
                        // k0 leading 1-byte codes, then (if it lies inside the window) one 2-byte code
                        const uint32_t k0  = hb ? uint32_t(__ffs(int(hb)) - 1) >> 3 : 4u;
                        const uint32_t k   = min(k0, rem);
                        const uint32_t x   = w >> (8u * (k & 3u));
                        bool           dbl = live && k0 < 3u && k0 < rem;
                        if (dbl && (x & 0xffu) >= 0xc0u) {
                                spill = true;
                                dbl   = false;
                        }
                        const uint32_t vd = ((x & 0x3fu) << 8) | ((x >> 8) & 0xffu);
                        const uint32_t np = live ? k + (dbl ? 1u : 0u) : 0u; // postings of this step (0..4)
                        const uint32_t r0 = rel + (np > 0u ? (k >= 1u ? b0 : vd) : 0u);
                        const uint32_t r1 = r0 + (np > 1u ? (k >= 2u ? b1 : vd) : 0u);
                        const uint32_t r2 = r1 + (np > 2u ? (k >= 3u ? b2 : vd) : 0u);
                        const uint32_t r3 = r2 + (np > 3u ? b3 : 0u);
                        own_add_if(bs, np > 0u && r0 < W, r0);
                        own_add_if(bs, np > 1u && r1 < W, r1);
                        own_add_if(bs, np > 2u && r2 < W, r2);
                        own_add_if(bs, np > 3u && r3 < W, r3);
                        rel = r3;
                        i += np;
                        sp += live ? k + (dbl ? 2u : 0u) : 0u;
                }
        }
        if (i < nd) {
                const uint8_t *g = index + off + (sp - base);
                for (; i < nd; ++i) {
                        rel += varbyte_get(g);
                        if (rel < W)
                                bs.add(rel);
                }
        }
        if (last - lo < W)
                bs.add(last - lo);
}

// Per-lane decoder into an OwnAcc — no votes: every lane walks ITS block through 32-bit windows of its gather slot, four 1-byte codes per
// window when it can, else up to two codes of 1-2 bytes (two such codes always fit a window); a longer code sends the lane to global
// memory for the rest of the block.  Used where the lanes of a group belong to different lists (flat-tree plans: there the
// warp-voted decoder above paying its one-code-per-step path for the whole warp whenever ONE lane holds a 2-byte code): a lane in a
// sparse list then costs the lanes in dense lists an idle step, not a slow step.
// `past`: 2^31 - W when every docID of the source is below 2^31 (a docID relative to the tile start in [W, 2^31) then lies BEHIND the tile
// and the rest of the block with it: a rare term's block straddles many tiles, its lane leaves the walk there), else 0 (never).
__device__ __forceinline__ void google_block_docs_lane(const uint8_t *__restrict__ index, uint32_t off, const uint8_t *buf, int lane, uint32_t n, uint32_t prev,
                                                       uint32_t last, uint32_t lo, uint32_t W, OwnAcc &bs, uint32_t past) {
        const uint32_t mis  = off & 15u;
        const uint32_t base = uint32_t(__cvta_generic_to_shared(buf + lane * kGatherBytes)) + mis; // shared address of the first delta byte
        const uint32_t nd   = n - 1u;
        uint32_t       sp = base, rel = prev - lo, i = 0;
        while (i < nd) {
                const uint32_t a = sp & ~3u;
                const uint32_t w = __funnelshift_r(lds_u32(a), lds_u32(a + 4u), (sp & 3u) * 8u); // bytes sp .. sp+3
                if ((w & 0x80808080u) == 0u && i + 4u <= nd) {
                        const uint32_t r0 = rel + (w & 0xffu), r1 = r0 + __byte_perm(w, 0u, 0x4441u), r2 = r1 + __byte_perm(w, 0u, 0x4442u), r3 = r2 + (w >> 24);
                        rel = r3;
                        sp += 4u;
                        i += 4u;
                        if (r0 < W && r3 < W) {
                                bs.add(r0);
                                bs.add(r1);
                                bs.add(r2);
                                bs.add(r3);
                        } else {
                                if (r0 < W) bs.add(r0);
                                if (r1 < W) bs.add(r1);
                                if (r2 < W) bs.add(r2);
                                if (r3 < W) bs.add(r3);
                        }
                        continue;
                }
                const uint32_t b0 = w & 0xffu;
                if (b0 >= 0xc0u)
                        break; // 3..5-byte code: the section may leave the slot
                const uint32_t two = b0 >> 7;
                uint32_t       len = 1u + two;
                rel += two ? (((b0 & 0x3fu) << 8) | __byte_perm(w, 0u, 0x4441u)) : b0;
                if (rel < W)
                        bs.add(rel);
                ++i;
                const uint32_t w2 = w >> (8u * len), c0 = w2 & 0xffu;
                if (i < nd && c0 < 0xc0u) { // the second code of the window
                        const uint32_t two2 = c0 >> 7;
                        rel += two2 ? (((c0 & 0x3fu) << 8) | ((w2 >> 8) & 0xffu)) : c0;
                        if (rel < W)
                                bs.add(rel);
                        ++i;
                        len += 1u + two2;
                }
                sp += len;
                if (rel - W < past)
                        return; // behind the tile (its last docID too)
        }
        if (i < nd) {
                const uint8_t *g = index + off + (sp - base);
                for (; i < nd; ++i) {
                        rel += varbyte_get(g);
                        if (rel < W)
                                bs.add(rel);
                }
        }
        if (last - lo < W)
                bs.add(last - lo);
}

// generic sinks (BitSink of the step programs, BitAcc of flat disjunctions): the byte-wise decoder over the lane's gather slot
template <class SINK>
__device__ __forceinline__ void google_block_docs_gather(unsigned, const uint8_t *__restrict__ index, uint32_t off, const uint8_t *buf, int lane, uint32_t n,
                                                         uint32_t prev, uint32_t last, uint32_t lo, uint32_t W, SINK &bs) {
        google_block_docs_bytes(index, off, buf, lane, n, prev, last, lo, W, bs);
}

// Decode blocks [bA, bB] of a Google term into the warp's bitmap.  `sparse`: the destination docset holds few candidates — check each
// block's docID range against it first and skip blocks (and whole groups) without candidates.
__device__ void google_leaf_warp(const DevIndex &ix, const DevTerm &T, uint32_t bA, uint32_t bB, uint32_t lo, uint32_t hi, BitSink &bs, const uint32_t *skipfilt,
                                 uint8_t *stage, uint32_t stageBytes, int lane) {
        const uint32_t *bl = ix.blk_last + T.dir_begin;
        const uint32_t *bo = ix.blk_off + T.dir_begin;
        // decode the blocks whose indices are given per lane (b valid where `need`)
        auto decode_group = [&](uint32_t b, bool need) {
                uint32_t off = 0, last = 0, prev = 0, n = 0;
                if (need) {
                        off  = bo[b];
                        last = bl[b];
                        prev = b ? bl[b - 1] : 0u;
                        n    = (b + 1u == T.nblocks) ? (T.documents - 32u * (T.nblocks - 1u)) : 32u;
                }
                const uint32_t needMask = __ballot_sync(0xffffffffu, need);
                if (needMask) {
                        gather_issue(ix.index, off, need, stage, lane);
                        gather_wait<0>();
                        if (need)
                                google_block_docs_gather(needMask, ix.index, off, stage, lane, n, prev, last, lo, hi - lo, bs);
                }
                __syncwarp();
        };
        if (!skipfilt) {
                for (uint32_t g = bA; g <= bB; g += 32u) {
                        const uint32_t b = g + uint32_t(lane);
                        decode_group(b, b <= bB);
                }
        } else {
                // Sparse destination docset (few candidates): first collect the blocks whose docID range still holds a candidate — the
                // advance()/skiplist step of the reference (google_codec.cpp:821-934) — THEN decode them 32 at a time.  Decoding inside the
                // scan loop ran the lane-serial block decoder with a few of 32 lanes active, which cost as many issue slots
                // as all the dense tiles together.
                uint32_t *     list = reinterpret_cast<uint32_t *>(stage + kGatherBufBytes); // behind the first gather buffer
                const uint32_t cap  = (stageBytes - kGatherBufBytes) / 4u - 32u;
                uint32_t       nlist = 0;
                auto           drain = [&]() {
                        __syncwarp();
                        for (uint32_t i0 = 0; i0 < nlist; i0 += 32u) {
                                const uint32_t idx = i0 + uint32_t(lane);
                                const bool     on  = idx < nlist;
                                decode_group(on ? list[idx] : 0u, on);
                        }
                        nlist = 0;
                        __syncwarp();
                };
                for (uint32_t g = bA; g <= bB; g += 32u) {
                        const uint32_t b    = g + uint32_t(lane);
                        bool           need = b <= bB;
                        if (need) {
                                const uint32_t last = bl[b], prev = b ? bl[b - 1] : 0u;
                                const uint32_t d0 = max(prev + 1u, lo), d1 = min(last, hi - 1u);
                                if (d1 < d0)
                                        need = false;
                                else {
                                        const uint32_t r0 = d0 - lo, r1 = d1 - lo, w0 = r0 >> 5, w1 = r1 >> 5;
                                        if (w1 - w0 <= 7u) {
                                                uint32_t any = 0;
                                                for (uint32_t w = w0; w <= w1; ++w) {
                                                        uint32_t m = skipfilt[w];
                                                        if (w == w0)
                                                                m &= 0xffffffffu << (r0 & 31u);
                                                        if (w == w1)
                                                                m &= 0xffffffffu >> (31u - (r1 & 31u));
                                                        any |= m;
                                                }
                                                need = any != 0;
                                        }
                                }
                        }
                        const uint32_t mask = __ballot_sync(0xffffffffu, need);
                        if (need)
                                list[nlist + __popc(mask & ((1u << lane) - 1u))] = b;
                        nlist += __popc(mask);
                        if (nlist > cap)
                                drain();
                }
                if (nlist)
                        drain();
        }
        bs.flush();
}

// LUCENE leaf: the blocks [bA, bB] of a term into the sink, one 128-document block at a time per warp (lucene_codec.cpp:515-594 refill_documents
// + FastPFor<4> __decodeArray fastpfor.h:222-270; block skipping == Decoder::advance's skiplist step, lucene_codec.cpp:596-656).
//   * 32 blocks are examined at once (lane = block): which of them can hold a document of the tile that the filter still wants;
//   * a needed block's bytes arrive by ONE 1-D bulk copy (cp.async.bulk + mbarrier, issued by lane 0) — and the NEXT needed block's copy is
//     issued as soon as the current block's values sit in registers, so it travels while the prefix sum runs and the bits are set
//     (a single staging buffer: a second one would cost resident warps);
//   * the page is unpacked vertically (lane l owns values l, l+32, l+64, l+96: lucene_intblock_v of score_flat.cuh), the freq int-block
//     behind it is never touched in DocumentsOnly mode.
// SINK: how a document reaches the bitmap (uniform per call, so decided once): 0 = or-in, 1 = or-in when the filter bitmap holds it (AND),
// 2 = clear when set (AND NOT)
template <int SINK>
__device__ void lucene_leaf_warp_t(const DevIndex &ix, const DevTerm &T, uint32_t bA, uint32_t bB, uint32_t lo, uint32_t hi, BitSink &bs, const uint32_t *skipfilt,
                                   uint8_t *stage, int lane, uint32_t bar_s, uint32_t &seq) {
        const uint32_t *const fw = SINK == 2 ? bs.bm : bs.filt; // the words a document is tested against (SINK 0: none)
        const uint32_t *bl      = ix.blk_last + T.dir_begin;
        const uint32_t *bo      = ix.blk_off + T.dir_begin;
        const uint32_t  nfull   = T.documents >> 7;
        const uint32_t  stage_s = uint32_t(__cvta_generic_to_shared(stage));
        uint32_t *      scratch = reinterpret_cast<uint32_t *>(stage + kGatherBufBytes);
        const uint32_t  W       = hi - lo; // (hi wraps to 0 only for the last tile of a 2^32 docID space: hi - lo is still the tile size)
        for (uint32_t b0 = bA; b0 <= bB; b0 += 32u) {
                // ---- lane = block b0 + lane: its bytes, its docID range, and whether the tile / the filter needs it
                const uint32_t b    = b0 + uint32_t(lane);
                bool           need = b <= bB;
                uint32_t       off = 0, offn = 0, prev = 0;
                if (need) {
                        off  = __ldg(bo + b);
                        offn = __ldg(bo + b + 1u);
                        prev = b ? __ldg(bl + b - 1u) : 0u;
                        const uint32_t last = __ldg(bl + b);
                        const uint32_t d0 = max(prev + 1u, lo), d1 = min(last - lo, W - 1u) + lo; // documents of the block inside the tile
                        if (last < lo || d1 < d0)
                                need = false;
                        else if (skipfilt) {
                                const uint32_t r0 = d0 - lo, r1 = d1 - lo, w0 = r0 >> 5, w1 = r1 >> 5;
                                if (w1 - w0 <= 15u) { // (a block spanning more of the tile than that is simply decoded)
                                        uint32_t any = 0;
                                        for (uint32_t w = w0; w <= w1; ++w) {
                                                uint32_t m = skipfilt[w];
                                                if (w == w0)
                                                        m &= 0xffffffffu << (r0 & 31u);
                                                if (w == w1)
                                                        m &= 0xffffffffu >> (31u - (r1 & 31u));
                                                any |= m;
                                        }
                                        need = any != 0u;
                                }
                        }
                }
                uint32_t mask = __ballot_sync(0xffffffffu, need);
                auto issue = [&](uint32_t j) { // bulk copy of lane j's block into the staging buffer
                        const uint32_t o = __shfl_sync(0xffffffffu, off, int(j)), on = __shfl_sync(0xffffffffu, offn, int(j));
                        const uint32_t abase = o & ~15u, bytes = min(((on + 15u) & ~15u) - abase, kGatherBufBytes);
                        if (lane == 0) {
                                mbar_expect_tx(bar_s, bytes);
                                bulk_g2s(stage_s, ix.index + abase, bytes, bar_s);
                        }
                };
                if (mask)
                        issue(uint32_t(__ffs(int(mask)) - 1));
                while (mask) {
                        const uint32_t j = uint32_t(__ffs(int(mask)) - 1);
                        mask &= mask - 1u;
                        const uint32_t bj = b0 + j, oj = __shfl_sync(0xffffffffu, off, int(j)), onj = __shfl_sync(0xffffffffu, offn, int(j));
                        const uint32_t pj = __shfl_sync(0xffffffffu, prev, int(j));
                        mbar_wait(bar_s, seq & 1u);
                        ++seq;
                        const uint32_t skew = oj & 15u;
                        if (bj < nfull) {
                                uint32_t d[4], dbits;
                                (void)lucene_intblock_v(stage, skew, lane, d, scratch, dbits);
                                __syncwarp(); // every lane has read the staging buffer: the next block may land in it
                                if (mask)
                                        issue(uint32_t(__ffs(int(mask)) - 1));
                                // docIDs = prev + inclusive prefix sum over the block (update_curdoc, lucene_codec.cpp:568-594), group by group
                                if (dbits <= 11u) { // 32 values below 2048 sum to less than 65536: two groups share one scan
                                        const uint32_t sa = warp_incl_scan(d[0] | (d[1] << 16), lane), sb = warp_incl_scan(d[2] | (d[3] << 16), lane);
                                        const uint32_t ta = __shfl_sync(0xffffffffu, sa, 31), tb = __shfl_sync(0xffffffffu, sb, 31);
                                        const uint32_t b1 = pj + (ta & 0xffffu), b2 = b1 + (ta >> 16), b3 = b2 + (tb & 0xffffu);
                                        d[0] = pj + (sa & 0xffffu);
                                        d[1] = b1 + (sa >> 16);
                                        d[2] = b2 + (sb & 0xffffu);
                                        d[3] = b3 + (sb >> 16);
                                } else {
                                        uint32_t base = pj;
#pragma unroll
                                        for (int g = 0; g < 4; ++g) {
                                                const uint32_t sc = warp_incl_scan(d[g], lane);
                                                d[g]              = base + sc;
                                                base += __shfl_sync(0xffffffffu, sc, 31);
                                        }
                                }
                                // the lane's four documents sit 32 documents apart (vertical layout): nothing to merge per lane, so they go straight
                                // into the sink's bitmap — the (up to) four filter / target words are loaded side by side first, and only a
                                // document the filter still wants costs an atomic
                                uint32_t rel[4], f[4];
#pragma unroll
                                for (int g = 0; g < 4; ++g) {
                                        rel[g] = d[g] - lo;
                                        if (SINK == 0)
                                                f[g] = rel[g] < W ? 0xffffffffu : 0u;
                                        else
                                                f[g] = rel[g] < W ? fw[rel[g] >> 5] : 0u;
                                }
#pragma unroll
                                for (int g = 0; g < 4; ++g) {
                                        const uint32_t bit = 1u << (rel[g] & 31u);
                                        if (f[g] & bit) {
                                                if (SINK == 2)
                                                        atomicAnd(&bs.bm[rel[g] >> 5], ~bit);
                                                else
                                                        atomicOr(&bs.bm[rel[g] >> 5], bit);
                                        }
                                }
                        } else {
                                // the term's tail: (varbyte delta, varbyte freq) pairs (lucene_codec.cpp:527-550), at most 127 of them
                                const uint32_t tail = T.documents & 127u;
                                const bool     fits = ((onj + 15u) & ~15u) - (oj & ~15u) <= kGatherBufBytes; // (10 bytes per pair at most: 1285 > the buffer never happens, but stay safe)
                                if (lane == 0) {
                                        const uint8_t *p   = fits ? stage + skew : ix.index + oj;
                                        uint32_t       doc = pj;
                                        for (uint32_t i = 0; i < tail; ++i) {
                                                doc += varbyte_get(p);
                                                (void)varbyte_get(p);
                                                if (doc - lo >= W && doc >= lo)
                                                        break;
                                                if (doc - lo < W)
                                                        bs.add(doc - lo);
                                        }
                                }
                                __syncwarp();
                                if (mask)
                                        issue(uint32_t(__ffs(int(mask)) - 1));
                        }
                }
        }
        bs.flush();
}
__device__ __forceinline__ void lucene_leaf_warp(const DevIndex &ix, const DevTerm &T, uint32_t bA, uint32_t bB, uint32_t lo, uint32_t hi, BitSink &bs,
                                                 const uint32_t *skipfilt, uint8_t *stage, int lane, uint32_t bar_s, uint32_t &seq) {
        if (bs.mode == M_ANDNOT)
                lucene_leaf_warp_t<2>(ix, T, bA, bB, lo, hi, bs, skipfilt, stage, lane, bar_s, seq);
        else if (bs.filt)
                lucene_leaf_warp_t<1>(ix, T, bA, bB, lo, hi, bs, skipfilt, stage, lane, bar_s, seq);
        else
                lucene_leaf_warp_t<0>(ix, T, bA, bB, lo, hi, bs, skipfilt, stage, lane, bar_s, seq);
}

#include "exec_docs_flat.cuh"
#include "exec_docs_cand.cuh"

// min 7 CTAs/SM: shared memory allows 7 at the default tile; without the bound ptxas stops at 64 registers and spills
// TREE: the flat-tree launch (every query of its ticket space is a flat-tree plan) — that instantiation holds nothing but the tree
// executor, and the other one does not carry it (the tree state lives in registers across the tile loop: in one kernel with the
// candidate and flat paths it pushed them over the 72-register bound)
// LUC: the launch runs over a LUCENE index (the codec is a property of the uploaded index, so of the launch): that instantiation carries the
// bulk-copy block decoder and none of the GOOGLE-only paths (candidate-driven, flat, flat-tree), and the GOOGLE ones do not carry it
template <bool PH, bool TREE, bool LUC> __global__ void __launch_bounds__(kDocsWarps * 32, PH ? 4 : (TREE ? 6 : 7)) k_exec_docs(ExecParams P) { // PH: see k_exec_tiles
        __shared__ __align__(8) unsigned long long s_lbar[kDocsWarps]; // LUCENE: one mbarrier per warp for its block copies
        uint32_t lseq = 0;                                            // ... and how many copies the warp has consumed (phase parity)
        if constexpr (LUC) {
                if ((threadIdx.x & 31) == 0) {
                        mbar_init(uint32_t(__cvta_generic_to_shared(&s_lbar[threadIdx.x >> 5])), 1);
                        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
                }
                __syncthreads();
        }
        const uint32_t W  = 1u << P.exec_shift;
        const uint32_t NW = W >> 5;
        const int      lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        const size_t   perWarp = size_t(P.nslots) * NW * 4 + P.docs_stage_bytes;
        uint32_t *     slots = reinterpret_cast<uint32_t *>(dyn_smem + perWarp * warp);
        uint8_t *      stage = reinterpret_cast<uint8_t *>(slots + size_t(P.nslots) * NW);
        const uint32_t wpl   = NW >> 5; // bitmap words per lane (contiguous ownership: lane l owns words [l*wpl, (l+1)*wpl))

        uint32_t curq = 0xffffffffu, qgen = 0; // qgen: the current query's first ticket
        DevQuery Q;
        Q.item_base = 0;
        Q.ntiles    = 0;
        TreeState TS; // flat-tree plans: the current query's leaves and slot operations, in lane registers
        TS.nleaf = TS.nops = 0;

        for (;;) {
                // tickets run over THIS launch's queries only (a batch can take two launches: trees on the flat-tree path use a smaller tile)
                uint32_t gitem = 0;
                if (lane == 0)
                        gitem = atomicAdd(P.ticket, 1u);
                gitem = __shfl_sync(0xffffffffu, gitem, 0);
                if (gitem >= P.gen_items)
                        break;
                if (curq == 0xffffffffu || gitem < qgen || gitem - qgen >= Q.ntiles) {
                        uint32_t qlo = 0, qhi = P.nq;
                        while (qhi - qlo > 1) {
                                const uint32_t mid = (qlo + qhi) >> 1;
                                const uint32_t gb  = P.gen_sel ? P.queries[mid].gen_base2 : P.queries[mid].gen_base;
                                if (gb <= gitem) qlo = mid;
                                else qhi = mid;
                        }
                        curq = qlo;
                        Q    = P.queries[qlo];
                        qgen = P.gen_sel ? Q.gen_base2 : Q.gen_base;
                        if constexpr (TREE)
                                tree_load(P, Q, TS, lane);
                }
                const uint32_t item = Q.item_base + (gitem - qgen); // batch-wide (query, tile) item: index of the segment arrays
                if constexpr (!TREE && !LUC) {
                        if (Q.route == TRN_ROUTE_CANDIDATE) { // candidate-driven conjunction: the work item is a 32-block group of the lead term
                                __syncwarp();
                                cand_exec_google(P, Q, curq, item, item - Q.item_base, slots, lane);
                                continue;
                        }
                }
                const uint32_t tile = Q.tile_lo + (item - Q.item_base);
                const uint32_t lo = tile << P.exec_shift, hi = lo + W;
                bool           dead = false;
                int            handled = 0;
                if constexpr (TREE) { // flat-tree plan: its leaves in (at most) two decode passes, then its slot operations
                        handled = tree_exec_google(P, Q, TS, lo, W, NW, slots, stage, lane) ? 2 : 1;
                } else if (!LUC && Q.route != TRN_ROUTE_STEPS) // (the flat AND / OR plans: the other routes never reach this launch)
                        handled = flat_exec_google(P, Q, lo, W, NW, slots, stage, lane);
                if (handled == 2)
                        dead = true;

                for (uint32_t si = 0; !TREE && si < Q.nsteps && !dead && handled == 0; ++si) {
                        const DevStep st  = P.steps[Q.step_begin + si];
                        uint32_t *    dst = slots + size_t(st.dst) * NW;
                        __syncwarp();
                        if (st.op == OP_CLEAR) {
                                for (uint32_t i = lane; i < NW; i += 32)
                                        dst[i] = 0;
                        } else if (st.op == OP_SLOT) {
                                const uint32_t *src = slots + size_t(st.src) * NW;
                                for (uint32_t i = lane; i < NW; i += 32) {
                                        const uint32_t s = src[i];
                                        if (st.mode == M_SET) dst[i] = s;
                                        else if (st.mode == M_OR) dst[i] |= s;
                                        else if (st.mode == M_AND) dst[i] &= s;
                                        else if (st.mode == M_ANDNOT) dst[i] &= ~s;
                                }
                        } else if (st.op == OP_COUNT_ADD) {
                                // bit-sliced saturating counters: plane j of the counter lives in slot dst + j
                                const uint32_t *src = slots + size_t(st.src) * NW;
                                for (uint32_t i = lane; i < NW; i += 32) {
                                        uint32_t carry = src[i];
                                        for (uint32_t j = 0; j < st.mode && carry; ++j) {
                                                uint32_t *     pl = slots + size_t(st.dst + j) * NW;
                                                const uint32_t p  = pl[i];
                                                pl[i]             = p ^ carry;
                                                carry &= p;
                                        }
                                        if (carry) // overflow: stay at the maximum
                                                for (uint32_t j = 0; j < st.mode; ++j)
                                                        slots[size_t(st.dst + j) * NW + i] |= carry;
                                }
                        } else if (st.op == OP_COUNT_GE) {
                                const uint32_t m = st.term;
                                for (uint32_t i = lane; i < NW; i += 32) {
                                        uint32_t gt = 0, eq = 0xffffffffu;
                                        for (int j = int(st.mode) - 1; j >= 0; --j) {
                                                const uint32_t p = slots[size_t(st.src + j) * NW + i];
                                                if ((m >> j) & 1u) eq &= p;
                                                else gt |= eq & p;
                                        }
                                        dst[i] = gt | eq;
                                }
                        } else if (st.op == OP_PHRASE) {
                                if constexpr (PH)
                                        phrase_check(P.ix, P.steps + Q.step_begin + si + 1u, st.mode, lo, NW, dst, nullptr, 0.0, lane, 32); // phrase.cuh
                        } else if (st.op == OP_LEAF && st.mode != M_NONE) {
                                uint32_t *tmp      = slots + size_t(P.nslots - 1) * NW;
                                const int mode     = st.mode;
                                const bool haveTerm = st.term != kEmptyTerm;
                                DevTerm    T;
                                uint32_t   bA = 1, bB = 0;
                                if (haveTerm) {
                                        T = P.ix.terms[st.term];
                                        tile_block_range(P.ix, T, lo, W, bA, bB);
                                }
                                const uint32_t *skipfilt = nullptr;
                                BitSink         bs;
                                // Google operands that are decoded in full go through the plain-store word builder into a bitmap of their
                                // own (dst itself for SET, the scratch slot otherwise) and are combined word-wise afterwards
                                const bool ownOk = !LUC && haveTerm && bA <= bB;
                                const uint32_t dummy = uint32_t(__cvta_generic_to_shared(stage + kGatherBufBytes)) + uint32_t(lane) * 4u;
                                if (ownOk && mode != M_AND) {
                                        uint32_t *out = mode == M_SET ? dst : tmp;
                                        bool      full = true;
                                        if (mode == M_ANDNOT) { // few documents left to exclude from: block skipping (below) beats a full decode
                                                uint32_t cnt = 0;
                                                for (uint32_t i = lane; i < NW; i += 32)
                                                        cnt += __popc(dst[i]);
                                                for (int d = 16; d > 0; d >>= 1)
                                                        cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
                                                full = cnt >= 4u * (bB - bA + 1u);
                                        }
                                        if (full) {
                                                for (uint32_t i = lane; i < NW; i += 32)
                                                        out[i] = 0;
                                                __syncwarp();
                                                google_leaf_own(P.ix, T, bA, bB, lo, W, out, stage, dummy, lane);
                                                if (mode == M_OR)
                                                        for (uint32_t i = lane; i < NW; i += 32)
                                                                dst[i] |= tmp[i];
                                                else if (mode == M_ANDNOT)
                                                        for (uint32_t i = lane; i < NW; i += 32)
                                                                dst[i] &= ~tmp[i];
                                                goto leaf_done;
                                        }
                                }
                                if (mode == M_SET) {
                                        for (uint32_t i = lane; i < NW; i += 32)
                                                dst[i] = 0;
                                        bs.init(dst, nullptr, M_OR);
                                } else if (mode == M_OR) {
                                        bs.init(dst, nullptr, M_OR);
                                } else if (mode == M_ANDNOT) {
                                        bs.init(dst, nullptr, M_ANDNOT);
                                        skipfilt = dst;
                                } else { // M_AND
                                        // candidates alive in dst: count + span (the GPU form of "where would advance() land")
                                        uint32_t cnt = 0, mn = 0xffffffffu, mx = 0;
                                        for (uint32_t i = 0; i < wpl; ++i) {
                                                const uint32_t wi = lane * wpl + i, w = dst[wi];
                                                tmp[wi]           = 0;
                                                if (w) {
                                                        cnt += __popc(w);
                                                        mn = min(mn, wi * 32u + uint32_t(__ffs(int(w)) - 1));
                                                        mx = wi * 32u + uint32_t(31 - __clz(int(w)));
                                                }
                                        }
                                        for (int d = 16; d > 0; d >>= 1) {
                                                cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
                                                mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, d));
                                                mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
                                        }
                                        if (cnt == 0) {
                                                bA = 1;
                                                bB = 0;
                                        } else if (ownOk && cnt >= kSparseThreshold) {
                                                // dense destination: full decode into the (just cleared) scratch slot, then one word-wise AND
                                                __syncwarp();
                                                google_leaf_own(P.ix, T, bA, bB, lo, W, tmp, stage, dummy, lane);
                                                for (uint32_t i = lane; i < NW; i += 32)
                                                        dst[i] &= tmp[i];
                                                goto leaf_done;
                                        } else if (cnt < kSparseThreshold && bA <= bB) {
                                                const uint32_t *bl = P.ix.blk_last + T.dir_begin;
                                                const uint32_t  a  = warp_lower_bound(bl, bA, bB, lo + mn, lane);
                                                if (a > bB) {
                                                        bA = 1;
                                                        bB = 0;
                                                } else {
                                                        const uint32_t b = warp_lower_bound(bl, a, bB, lo + mx, lane);
                                                        bA               = a;
                                                        bB               = min(b, bB);
                                                }
                                                skipfilt = dst;
                                        }
                                        bs.init(tmp, dst, M_OR);
                                }
                                __syncwarp();
                                if (haveTerm && bA <= bB) {
                                        if constexpr (!LUC)
                                                google_leaf_warp(P.ix, T, bA, bB, lo, hi, bs, skipfilt, stage, P.docs_stage_bytes, lane);
                                        else
                                                lucene_leaf_warp(P.ix, T, bA, bB, lo, hi, bs, skipfilt, stage, lane, uint32_t(__cvta_generic_to_shared(&s_lbar[warp])), lseq);
                                }
                                if (mode == M_AND) {
                                        __syncwarp();
                                        for (uint32_t i = lane; i < NW; i += 32)
                                                dst[i] = tmp[i];
                                }
                        leaf_done:;
                        }
                        if (st.flags & F_BREAK_IF_EMPTY) {
                                __syncwarp();
                                uint32_t any = 0;
                                for (uint32_t i = lane; i < NW; i += 32)
                                        any |= dst[i];
                                if (!__any_sync(0xffffffffu, any != 0))
                                        dead = true;
                        }
                }
                __syncwarp();

                // ---- masked documents (docidupdates.h masked_documents_registry::test, exec.cpp:1108-1116) never reach the sink
                if (!dead && P.ix.masked) {
                        uint32_t *      r  = slots + size_t(Q.root_slot) * NW;
                        const uint32_t *mk = P.ix.masked + (lo >> 5);
                        for (uint32_t i = lane; i < NW; i += 32)
                                r[i] &= ~mk[i];
                        __syncwarp();
                }
                // ---- emission: ordered compaction of the root docset
                uint32_t c = 0, full = 0;
                const uint32_t *root = slots + size_t(Q.root_slot) * NW;
                if (!dead) {
                        uint32_t cb = 0; // documents of the current 256-docID bucket (8 words): 256 of them do not fit the bucketed form's count byte
                        for (uint32_t i = 0; i < wpl; ++i) {
                                const uint32_t pc = __popc(root[lane * wpl + i]);
                                c += pc;
                                cb += pc;
                                if ((i & 7u) == 7u) {
                                        full |= cb == 256u ? 1u : 0u;
                                        cb = 0;
                                }
                        }
                }
                const uint32_t incl  = warp_incl_scan(c, lane);
                const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
                unsigned long long base = 0;
                if (P.item_desc) {
                        // ---- compact results, whichever form takes the fewest words (a tile holds at most 2^16 documents):
                        //   bitmap   the tile's words                                                          dense tiles (> 1 document in 8)
                        //   U8B      per 256-docID bucket a count byte, then one offset byte per document      1 in 8 .. 1 in 256
                        //   U16      16-bit offsets from the tile's first docID, two per word                  sparse tiles
                        const uint32_t nbk  = W >> 8;
                        const bool     u8ok = wpl >= 8u && W <= 65536u && !__any_sync(0xffffffffu, full != 0u); // a lane owns whole buckets
                        uint32_t       enc = kEncBitmap, words = NW;
                        if (W <= 65536u) {
                                if (((total + 1u) >> 1) < words)
                                        enc = kEncU16, words = (total + 1u) >> 1;
                                if (u8ok && ((nbk + total + 3u) >> 2) < words)
                                        enc = kEncU8B, words = (nbk + total + 3u) >> 2;
                        }
                        if (!total)
                                words = 0;
                        if (lane == 0) {
                                if (total) {
                                        base = atomicAdd(P.seg_cursor, static_cast<unsigned long long>(words));
                                        atomicAdd(&P.match_counts[curq], static_cast<unsigned long long>(total));
                                        atomicAdd(&P.word_counts[curq], static_cast<unsigned long long>(words));
                                        if (base + words > P.seg_capacity) {
                                                *P.overflow = 1;
                                                base        = ~0ull;
                                        }
                                }
                                P.item_off[item]  = base;
                                P.item_cnt[item]  = base == ~0ull ? 0u : words;
                                P.item_desc[item] = base == ~0ull ? 0u : (total | enc << 30);
                        }
                        base = __shfl_sync(0xffffffffu, base, 0);
                        if (total && base != ~0ull) {
                                if (enc == kEncBitmap) {
                                        for (uint32_t i = lane; i < NW; i += 32)
                                                P.seg_docids[base + i] = root[i];
                                } else if (enc == kEncU8B) {
                                        uint8_t *o8  = reinterpret_cast<uint8_t *>(P.seg_docids + base);
                                        uint32_t pos = nbk + (incl - c), cb = 0;
                                        for (uint32_t i = 0; i < wpl; ++i) {
                                                const uint32_t wi = lane * wpl + i;
                                                uint32_t       w  = root[wi];
                                                cb += __popc(w);
                                                while (w) {
                                                        const uint32_t bit = uint32_t(__ffs(int(w)) - 1);
                                                        w &= w - 1;
                                                        o8[pos++] = uint8_t((wi & 7u) * 32u + bit);
                                                }
                                                if ((i & 7u) == 7u) {
                                                        o8[wi >> 3] = uint8_t(cb);
                                                        cb          = 0;
                                                }
                                        }
                                        if (lane == 31)
                                                for (uint32_t z = nbk + total; z < words * 4u; ++z)
                                                        o8[z] = 0; // the pad bytes travel too
                                } else {
                                        uint16_t *out = reinterpret_cast<uint16_t *>(P.seg_docids + base);
                                        uint32_t  pos = incl - c;
                                        for (uint32_t i = 0; i < wpl; ++i) {
                                                const uint32_t wi = lane * wpl + i;
                                                uint32_t       w  = root[wi];
                                                while (w) {
                                                        const uint32_t bit = uint32_t(__ffs(int(w)) - 1);
                                                        w &= w - 1;
                                                        out[pos++] = uint16_t(wi * 32u + bit);
                                                }
                                        }
                                        if (lane == 31 && (total & 1u))
                                                out[total] = 0; // the pad half-word travels too
                                }
                        }
                        continue;
                }
                if (lane == 0) {
                        if (total) {
                                base = atomicAdd(P.seg_cursor, static_cast<unsigned long long>(total));
                                atomicAdd(&P.match_counts[curq], static_cast<unsigned long long>(total));
                                if (base + total > P.seg_capacity) {
                                        *P.overflow = 1;
                                        base        = ~0ull;
                                }
                        }
                        P.item_off[item] = base;
                        P.item_cnt[item] = base == ~0ull ? 0u : total;
                }
                base = __shfl_sync(0xffffffffu, base, 0);
                if (total && base != ~0ull) {
                        unsigned long long pos = base + (incl - c);
                        for (uint32_t i = 0; i < wpl; ++i) {
                                const uint32_t wi = lane * wpl + i;
                                uint32_t       w  = root[wi];
                                while (w) {
                                        const uint32_t bit = uint32_t(__ffs(int(w)) - 1);
                                        w &= w - 1;
                                        P.seg_docids[pos++] = lo + wi * 32u + bit;
                                }
                        }
                }
        }
}

uint32_t exec_docs_cand_smem_bytes(bool with_membership) {
        return with_membership ? kCandSmemMask : kCandSmem;
}

uint32_t exec_docs_stage_bytes() {
        return kDocsStageBytes1;
}

size_t exec_docs_smem_bytes(uint32_t exec_shift, uint32_t nslots, uint32_t stageBytes) {
        const size_t NW = (size_t(1) << exec_shift) >> 5;
        return size_t(kDocsWarps) * (size_t(nslots) * NW * 4 + stageBytes);
}

int exec_docs_max_ctas_per_sm(uint32_t exec_shift, uint32_t nslots, uint32_t stageBytes, bool tree, bool lucene) {
        const size_t smem = exec_docs_smem_bytes(exec_shift, nslots, stageBytes);
        const void *fns[2];
        if (lucene) {
                fns[0] = (const void *)k_exec_docs<false, false, true>;
                fns[1] = (const void *)k_exec_docs<true, false, true>;
        } else if (tree) {
                fns[0] = fns[1] = (const void *)k_exec_docs<false, true, false>;
        } else {
                fns[0] = (const void *)k_exec_docs<false, false, false>;
                fns[1] = (const void *)k_exec_docs<true, false, false>;
        }
        int best = 0;
        for (int i = 0; i < 2; ++i) {
                if (cudaFuncSetAttribute(fns[i], cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess)
                        return 0;
                int n = 0;
                if (i == 0 && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fns[i], kDocsWarps * 32, smem) != cudaSuccess)
                        return 0;
                if (i == 0)
                        best = n;
        }
        return best;
}

cudaError_t launch_exec_docs(const ExecParams &P, int grid, cudaStream_t stream) {
        const size_t smem = exec_docs_smem_bytes(P.exec_shift, P.nslots, P.docs_stage_bytes);
        // gen_sel == 1: the flat-tree launch (its ticket space holds flat-tree plans only; phrase plans never take that path; GOOGLE only)
        const void *fn;
        if (P.ix.codec != 0)
                fn = P.has_phrase ? (const void *)k_exec_docs<true, false, true> : (const void *)k_exec_docs<false, false, true>;
        else
                fn = P.gen_sel ? (const void *)k_exec_docs<false, true, false>
                               : (P.has_phrase ? (const void *)k_exec_docs<true, false, false> : (const void *)k_exec_docs<false, false, false>);
        cudaError_t  e    = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
        if (e != cudaSuccess)
                return e;
        void *args[] = {(void *)&P};
        return cudaLaunchKernel(fn, dim3(grid), dim3(kDocsWarps * 32), args, smem, stream);
}
