// Candidate-driven conjunctions in k_exec_docs == the leap-frog of DocsSetIterators::Conjuction / ConjuctionAllPLI
// (docset_iterators.cpp:226-348: the rarest operand leads, every other operand advance()s to the lead's document) — used when the
// lead is SPARSE relative to the docID tiles of the bitmap path.  (Included by exec_docs.cuh.)
//
// Why: the bitmap path pays ~1500 warp-instructions per (query, 16384-doc tile) before it decodes anything (slot clears, the
// word-wise AND, count, emission), and a sparse operand contributes one or two blocks per tile, so most (query, tile) items of the
// 2-term AND workload are nearly empty groups at a few active lanes (most of
// the work items belong to queries whose rarest term has < 4 blocks per tile).  Here a work item is one GROUP OF 32 BLOCKS OF THE
// LEAD TERM, wherever its documents lie:
//   1. lane = block: the 32 blocks are decoded into a candidate array in shared memory (row stride 33 words: conflict-free for
//      the lane-per-block writes and for the lane-per-candidate reads below);
//   2. for every other operand, for each lead block (32 candidates, lane = candidate): the lane finds the one block of the operand
//      that can hold its candidate — the term's sparse docID -> block table bounds the block directory, a short binary search over
//      blk_last finishes it (== skiplist_search + the header hops of Decoder::advance, google_codec.cpp:821-934, in O(log) loads) —
//      stages that block's head with cp.async and decodes it only as far as the candidate;
//   3. the survivors (minus masked documents) are compacted and emitted in order.
// Cost is proportional to the LEAD's postings, not to the docID space, and no bitmap is touched.
#pragma once

static constexpr uint32_t kCandStride  = 33;
static constexpr uint32_t kCandWords   = 32 * kCandStride;      // 1056 words
static constexpr uint32_t kCandBytes   = kCandWords * 4;        // 4224 B (multiple of 16: the gather buffer follows)
static constexpr uint32_t kCandMaskBytes = kCandWords;            // one membership byte per candidate (terms that are not necessary)
static constexpr uint32_t kCandSmem    = kCandBytes + kGatherBufBytes;                  // candidates | one gather buffer
static constexpr uint32_t kCandSmemMask = kCandSmem + kCandMaskBytes;                   // ... | membership bytes (only queries with terms that are not necessary)
static constexpr uint32_t kCandInvalid = 0xffffffffu;
static constexpr uint32_t kCandProbeRounds = 2;                  // bitmap probes: rounds whose word loads are in flight together (at 4, k_exec_docs spills)
static_assert(32u % kCandProbeRounds == 0, "a group's 32 rounds split into whole batches");

// one lane decodes the doc section of ITS staged block into out[0..n).  Branch-free per code: the 32 lanes of a group hold blocks with
// different mixes of 1-, 2- and 3-byte codes, and a loop that branches on the code length (with early exits) does not reconverge before
// its end: such a loop ran at a few of 32 lanes.  Every lane runs the same 31 steps; a lane whose block ends, whose next
// code may leave its 80-byte slot or is longer than 3 bytes goes idle and finishes from global memory afterwards.
__device__ __forceinline__ void google_block_to_array(const uint8_t *__restrict__ index, uint32_t off, const uint8_t *buf, int lane, uint32_t n, uint32_t prev,
                                                      uint32_t last, uint32_t *out) {
        const uint32_t mis = off & 15u;
        const uint32_t sp  = uint32_t(__cvta_generic_to_shared(buf + lane * kGatherBytes)) + mis;
        const uint32_t nd  = n - 1u;
        uint32_t       doc = prev, i = 0, p = 0;
        bool           live = true;
#pragma unroll 1
        for (uint32_t it = 0; it < 31u; ++it) {
                const uint32_t at = sp + p, a = at & ~3u;
                const uint32_t w  = __funnelshift_r(lds_u32(a), lds_u32(a + 4u), (at & 3u) * 8u); // bytes p .. p+3 (reads stay inside the staging area)
                const uint32_t b0 = w & 0xffu;
                const uint32_t two = b0 >= 0x80u ? 1u : 0u, three = b0 >= 0xc0u ? 1u : 0u;
                const uint32_t v2 = ((b0 & 0x3fu) << 8) | ((w >> 8) & 0xffu), v3 = ((b0 & 0x1fu) << 16) | ((w >> 8) & 0xffffu);
                const uint32_t v  = three ? v3 : (two ? v2 : b0);
                // 3-byte codes (gaps >= 16384: the sparsest leads) are decoded in place too, so the 31 x 2 + 15 <= 80 bound of the other
                // decoders does not hold here: every code (<= 3 bytes) is checked against the end of the slot
                live = live && it < nd && b0 < 0xe0u && mis + p + 3u <= kGatherBytes;
                if (live) {
                        doc += v;
                        out[it] = doc;
                        p += 1u + two + three;
                        i = it + 1u;
                }
        }
        if (i < nd) {
                const uint8_t *g = index + off + p;
                for (; i < nd; ++i) {
                        doc += varbyte_get(g);
                        out[i] = doc;
                }
        }
        out[nd] = last;
}

// one lane walks ITS staged block until it reaches `target`; true if the block holds it (the block's last document is known
// from the directory and checked by the caller)
__device__ __forceinline__ bool google_block_find(const uint8_t *__restrict__ index, uint32_t off, const uint8_t *buf, int lane, uint32_t n, uint32_t prev,
                                                  uint32_t target) {
        const uint32_t mis = off & 15u;
        uint32_t       sp  = uint32_t(__cvta_generic_to_shared(buf + lane * kGatherBytes)) + mis;
        const uint32_t nd  = n - 1u;
        uint32_t       doc = prev, i = 0, p = 0;
        bool           spill = false;
        while (i < nd && !spill) {
                // four 1-byte codes at a time while their sum stays below the target (one dot product instead of four decode steps)
                while (i + 4u <= nd) {
                        const uint32_t a = (sp + p) & ~3u;
                        const uint32_t w = __funnelshift_r(lds_u32(a), lds_u32(a + 4u), ((sp + p) & 3u) * 8u);
                        if (w & 0x80808080u)
                                break;
                        const uint32_t sum = __dp4a(w, 0x01010101u, 0u);
                        if (doc + sum >= target)
                                break;
                        doc += sum;
                        p += 4u;
                        i += 4u;
                }
                for (uint32_t k = 0; k < 4u && i < nd; ++k, ++i) {
                        const uint32_t b0 = lds_u8(sp + p);
                        uint32_t       v;
                        if (b0 < 0x80u) {
                                v = b0;
                                p += 1u;
                        } else if (b0 < 0xc0u) {
                                v = ((b0 & 0x3fu) << 8) | lds_u8(sp + p + 1u);
                                p += 2u;
                        } else {
                                spill = true; // 3..5-byte code: the section may leave the slot
                                break;
                        }
                        doc += v;
                        if (doc >= target)
                                return doc == target;
                }
        }
        if (i < nd) {
                const uint8_t *g = index + off + p;
                for (; i < nd; ++i) {
                        doc += varbyte_get(g);
                        if (doc >= target)
                                return doc == target;
                }
        }
        return false;
}

// `cand`: kCandWords words, then one gather buffer, then (if the batch has such queries) kCandMaskBytes membership bytes.  `group`: 32-block group of the lead term.
// The query's program is [OP_LEAF lead, OP_LEAF term 1, ..., OP_TABLE x2]: terms 1 .. Q.root_slot-1 are NECESSARY (a candidate without
// them is dropped at once); the others only set their bit in the candidate's membership byte, and the truth table (bit m = value of
// the query when exactly the terms in m are present; bit 0 of m = the lead) decides at the end.
// FILT: the query may have a document filter (ExecParams::filters): a group wholly outside its allow set's span is skipped, and the
// filter drops documents beside the masked ones.
template <bool FILT> __device__ void cand_exec_google(const ExecParams &P, const DevQuery &Q, uint32_t curq, uint32_t item, uint32_t group, uint32_t *cand, int lane) {
        uint8_t *const stage = reinterpret_cast<uint8_t *>(cand + kCandWords);
        uint8_t *const cmask = stage + kGatherBufBytes;
        // lane j adopts the j-th term; lane w (< 8) keeps word w of the truth table
        uint32_t nleaf = 0, myTerm = kEmptyTerm, myTable = 0;
        for (uint32_t si = 0; si < Q.nsteps; ++si) {
                const DevStep st = P.steps[Q.step_begin + si];
                if (st.op == OP_LEAF) {
                        if (uint32_t(lane) == nleaf)
                                myTerm = st.term;
                        ++nleaf;
                } else if (st.op == OP_TABLE) {
                        const unsigned long long hi = static_cast<unsigned long long>(__double_as_longlong(st.idf));
                        const uint32_t           w  = uint32_t(lane) - st.dst; // 0..3 for the lanes that own these words
                        if (w == 0u) myTable = st.term;
                        else if (w == 1u) myTable = st.pad2;
                        else if (w == 2u) myTable = uint32_t(hi);
                        else if (w == 3u) myTable = uint32_t(hi >> 32);
                }
        }
        const uint32_t nnec = Q.root_slot; // necessary terms incl. the lead
        uint32_t mydir = 0, mynb = 0, mydocs = 0, myfirst = 0, mylast = 0, mytfb = 0, mytfbase = 0, mytfs = 32, mydense = kDenseNone;
        if (uint32_t(lane) < nleaf && myTerm != kEmptyTerm) {
                const DevTerm T = P.ix.terms[myTerm];
                if (P.ix.probe_off)
                        mydense = __ldg(P.ix.probe_off + myTerm);
                mydir           = T.dir_begin;
                mynb            = T.nblocks;
                mydocs          = T.documents;
                myfirst         = T.first_doc;
                mylast          = T.last_doc;
                mytfb           = T.tf_begin;
                mytfbase        = T.tf_base;
                mytfs           = T.tf_shift;
        }
        // ---- 1. the lead's blocks -> candidates
        const uint32_t dir0 = __shfl_sync(0xffffffffu, mydir, 0), nb0 = __shfl_sync(0xffffffffu, mynb, 0), docs0 = __shfl_sync(0xffffffffu, mydocs, 0);
        DevFilter      F{};
        if constexpr (FILT) {
                F = P.filters[curq];
                // the group's docIDs lie in (last docID of the block before it, last docID of its last block]
                const uint32_t b0 = group * 32u, b1 = min(nb0, b0 + 32u);
                const bool     out = b0 >= b1 || F.lo > F.hi || __ldg(P.ix.blk_last + dir0 + b1 - 1u) < F.lo || (b0 && __ldg(P.ix.blk_last + dir0 + b0 - 1u) >= F.hi);
                if (out) {
                        if (lane == 0) {
                                P.item_off[item] = 0;
                                P.item_cnt[item] = 0;
                                if (P.item_desc)
                                        P.item_desc[item] = 0;
                        }
                        return;
                }
        }
        uint32_t       n = 0;
        {
                const uint32_t b    = group * 32u + uint32_t(lane);
                const bool     have = b < nb0;
                uint32_t       off = 0, prev = 0, last = 0;
                if (have) {
                        const uint32_t *bl = P.ix.blk_last + dir0, *bo = P.ix.blk_off + dir0;
                        off  = bo[b];
                        last = bl[b];
                        prev = b ? bl[b - 1] : 0u;
                        n    = (b + 1u == nb0) ? (docs0 - 32u * (nb0 - 1u)) : 32u;
                }
                gather_issue(P.ix.index, off, have, stage, lane);
                gather_wait<0>();
                if (have)
                        google_block_to_array(P.ix.index, off, stage, lane, n, prev, last, cand + lane * kCandStride);
                __syncwarp();
        }
        const uint32_t rounds = min(32u, nb0 - min(nb0, group * 32u)); // lead blocks of this group (they are the leading lanes)
        if (nleaf > nnec) {
                for (uint32_t i = lane; i < kCandMaskBytes / 4u; i += 32)
                        reinterpret_cast<uint32_t *>(cmask)[i] = 0x01010101u; // bit 0: the lead holds every candidate
                __syncwarp();
        }
        // ---- 2. every other operand: keep the candidates it holds
        for (uint32_t t = 1; t < nleaf; ++t) {
                const uint32_t  dirt = __shfl_sync(0xffffffffu, mydir, int(t)), nbt = __shfl_sync(0xffffffffu, mynb, int(t)), docst = __shfl_sync(0xffffffffu, mydocs, int(t));
                const uint32_t  firstt = __shfl_sync(0xffffffffu, myfirst, int(t)), lastt = __shfl_sync(0xffffffffu, mylast, int(t));
                const uint32_t  tfbt = __shfl_sync(0xffffffffu, mytfb, int(t)), tfbaset = __shfl_sync(0xffffffffu, mytfbase, int(t)), tfst = __shfl_sync(0xffffffffu, mytfs, int(t));
                const uint32_t *bl = P.ix.blk_last + dirt, *bo = P.ix.blk_off + dirt;
                const uint32_t  denset = __shfl_sync(0xffffffffu, mydense, int(t));
                uint32_t        alive = 0;
                // round j's verdicts: a necessary term drops the candidates it does not hold, another one sets its membership bit
                auto keep = [&](uint32_t j, bool valid, bool hit) {
                        if (t < nnec) {
                                if (valid && !hit)
                                        cand[j * kCandStride + lane] = kCandInvalid;
                                alive |= __ballot_sync(0xffffffffu, valid && hit);
                        } else {
                                if (valid && hit)
                                        cmask[j * kCandStride + lane] |= uint8_t(1u << t);
                                alive = 1u;
                        }
                };
                if (denset != kDenseNone) {
                        // a term with a resident bitmap: the probe is one word load and a bit test.  The words of kR rounds are
                        // loaded before any of them is tested, so the group waits out one load latency per batch of rounds, not per round.
                        // (Lanes j >= rounds hold n = 0: the rounds past the group's blocks have no valid candidate.)  The filtered
                        // instantiation probes one round at a time: two rounds there add to the spills it already has.
                        const uint32_t *bmt   = P.ix.dense + denset;
                        const uint32_t  baset = (firstt >> kDenseAlignShift) << kDenseAlignShift;
                        constexpr uint32_t kR = FILT ? 1u : kCandProbeRounds;
                        for (uint32_t j0 = 0; j0 < rounds; j0 += kR) {
                                uint32_t w[kR], meta = 0; // meta bits 6r .. 6r + 5: round r's candidate is valid (bit 5), its bit in w[r]
#pragma unroll
                                for (uint32_t r = 0; r < kR; ++r) {
                                        const uint32_t nj = __shfl_sync(0xffffffffu, n, int(j0 + r));
                                        const uint32_t c  = uint32_t(lane) < nj ? cand[(j0 + r) * kCandStride + lane] : kCandInvalid;
                                        w[r]              = c != kCandInvalid && c >= firstt && c <= lastt ? __ldg(bmt + ((c - baset) >> 5)) : 0u;
                                        meta |= ((c != kCandInvalid ? 32u : 0u) | (c & 31u)) << (6u * r);
                                }
#pragma unroll
                                for (uint32_t r = 0; r < kR; ++r) {
                                        const uint32_t m     = (meta >> (6u * r)) & 63u;
                                        const bool     valid = m & 32u;
                                        if (__any_sync(0xffffffffu, valid))
                                                keep(j0 + r, valid, (w[r] >> (m & 31u)) & 1u);
                                }
                        }
                } else {
                        for (uint32_t j = 0; j < rounds; ++j) {
                                const uint32_t nj = __shfl_sync(0xffffffffu, n, int(j));
                                uint32_t       c  = uint32_t(lane) < nj ? cand[j * kCandStride + lane] : kCandInvalid;
                                const bool     valid = c != kCandInvalid;
                                if (!__any_sync(0xffffffffu, valid))
                                        continue;
                                bool     hit = false, need = false;
                                uint32_t off = 0, prev = 0, nblk = 0;
                                if (valid && nbt) {
                                        // the one block that can hold c: first block whose last document is >= c
                                        const uint32_t lo = first_block_ge(P.ix, dirt, nbt, firstt, lastt, tfbt, tfbaset, tfst, c);
                                        if (lo < nbt) {
                                                const uint32_t lastv = __ldg(bl + lo);
                                                if (lastv >= c) {
                                                        hit  = lastv == c;
                                                        need = !hit;
                                                        off  = __ldg(bo + lo);
                                                        prev = lo ? __ldg(bl + lo - 1u) : 0u;
                                                        nblk = (lo + 1u == nbt) ? (docst - 32u * (nbt - 1u)) : 32u;
                                                        if (need && c <= prev) // cannot happen (prev < c by construction); keeps a corrupt directory from looping
                                                                need = false;
                                                }
                                        }
                                }
                                if (__any_sync(0xffffffffu, need)) {
                                        gather_issue(P.ix.index, off, need, stage, lane);
                                        gather_wait<0>();
                                        if (need)
                                                hit = google_block_find(P.ix.index, off, stage, lane, nblk, prev, c);
                                        __syncwarp();
                                }
                                keep(j, valid, hit);
                        }
                }
                __syncwarp();
                if (!alive) {
                        // nothing survived this operand: the group matches nothing
                        if (lane == 0) {
                                P.item_off[item] = 0;
                                P.item_cnt[item] = 0;
                                if (P.item_desc)
                                        P.item_desc[item] = 0;
                        }
                        return;
                }
        }
        // ---- 3. masked documents, then ordered emission (lane j keeps the survivor mask of lead block j)
        uint32_t mymask = 0;
        for (uint32_t j = 0; j < rounds; ++j) {
                const uint32_t nj = __shfl_sync(0xffffffffu, n, int(j));
                const uint32_t c  = uint32_t(lane) < nj ? cand[j * kCandStride + lane] : kCandInvalid;
                bool           ok = c != kCandInvalid;
                if (nleaf > nnec) { // the membership bits of the terms that are not necessary decide (uniform shuffle: every lane takes part)
                        const uint32_t m    = ok ? (uint32_t(cmask[j * kCandStride + lane]) | ((1u << nnec) - 1u)) : 0u;
                        const uint32_t word = __shfl_sync(0xffffffffu, myTable, int(m >> 5));
                        ok                  = ok && ((word >> (m & 31u)) & 1u);
                }
                if (ok && P.ix.masked)
                        ok = ((__ldg(P.ix.masked + (c >> 5)) >> (c & 31u)) & 1u) == 0u;
                if constexpr (FILT) {
                        if (ok)
                                ok = (filter_keep(F, c >> 5) >> (c & 31u)) & 1u;
                }
                const uint32_t vm = __ballot_sync(0xffffffffu, ok);
                if (uint32_t(lane) == j)
                        mymask = vm;
        }
        const uint32_t cnt   = __popc(mymask);
        const uint32_t incl  = warp_incl_scan(cnt, lane);
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        unsigned long long base = 0;
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
                if (P.item_desc) { // compact results: a lead-block group is not a docID tile — plain docIDs (kEncU32), one word each
                        P.item_desc[item] = base == ~0ull ? 0u : total;
                        if (total)
                                atomicAdd(&P.word_counts[curq], static_cast<unsigned long long>(total));
                }
        }
        base = __shfl_sync(0xffffffffu, base, 0);
        if (!total || base == ~0ull)
                return;
        const uint32_t excl = incl - cnt;
        for (uint32_t j = 0; j < rounds; ++j) {
                const uint32_t vm = __shfl_sync(0xffffffffu, mymask, int(j));
                const uint32_t at = __shfl_sync(0xffffffffu, excl, int(j));
                if ((vm >> lane) & 1u)
                        P.seg_docids[base + at + __popc(vm & ((1u << lane) - 1u))] = cand[j * kCandStride + lane];
        }
}
