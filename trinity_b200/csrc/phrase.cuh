// Positions on the device (SURVEY.md 8f row 3) — GOOGLE codec: the inline hit streams of google_codec.cpp:533-594 (materialize_hits) and
// Phrase::consider_phrase_match (docset_iterators.cpp:66-158).  (Included by kernels.cu.)
//
// A phrase node "t0 t1 ... t(k-1)" is compiled (planner.cpp, Compiler::phrase_leaf) into
//     [OP_LEAF SET t(a) -> s] [OP_LEAF AND t(b) -> s] ...     the conjunction of its distinct terms: the documents that CAN match
//     [OP_PHRASE mode = k, dst = s, idf = sum of the terms' idf] [OP_ARG ...]       the position check, in place, over the survivors
// so the docset part runs on the existing leaf decoders (incl. their block skipping), and only the surviving candidates pay for positions.
// OP_PHRASE keeps a candidate d of slot s iff some non-zero position q of t0 has t(j) at q + j for every j; matchCnt = the number of such q
// (the Phrase scorer scores score(matchCnt, sum idf), docset_iterators_scorers.cpp:195-228).  One thread owns whole bitmap words, so the
// slot is filtered without atomics.  Per candidate and term a cursor walks the term's block straight from global memory: the doc deltas
// (to find the document's index in its block), the freqs (how many hits precede its own), the hits of the preceding documents, then its
// own positions — the skip_block_doc walk of google_codec.cpp:497-531.  Two cursors are alive at a time (t0 and t(j), merge-joined), the
// verdicts of up to 64 positions of t0 travel in a bit mask; documents with more hits of t0 are handled in chunks of 64.
#pragma once

// (the cursors themselves: hitcursor.h, shared with the host and included by kernels.cu ahead of namespace trn)
__device__ __forceinline__ PhraseTerm phrase_term(const DevIndex &ix, uint32_t term) {
        PhraseTerm    t;
        const DevTerm T = ix.terms[term];
        t.dir    = T.dir_begin;
        t.nb     = T.nblocks;
        t.docs   = T.documents;
        t.first  = T.first_doc;
        t.last   = T.last_doc;
        t.tfb    = T.tf_begin;
        t.tfbase = T.tf_base;
        t.tfs    = T.tf_shift;
        t.id     = term;
        return t;
}

// term id j of a phrase: four per OP_ARG step (term, pad2, idf as two words)
__device__ __forceinline__ uint32_t phrase_arg(const DevStep *args, uint32_t j) {
        const DevStep &a = args[j >> 2];
        const uint32_t s = j & 3u;
        if (s == 0u) return a.term;
        if (s == 1u) return a.pad2;
        const unsigned long long w = static_cast<unsigned long long>(__double_as_longlong(a.idf));
        return s == 2u ? uint32_t(w) : uint32_t(w >> 32);
}


__device__ __forceinline__ HitsView hits_view(const DevIndex &ix) {
        HitsView v;
        v.index      = ix.index;
        v.blk_last   = ix.blk_last;
        v.blk_off    = ix.blk_off;
        v.tile_first = ix.tile_first;
        v.hits       = ix.hits;
        v.hit_base   = ix.hit_base;
        v.hblk_off   = ix.hblk_off;
        v.hit_term   = ix.hit_term;
        v.codec      = ix.codec;
        return v;
}

// number of non-zero positions q of t0 in document d with t(j) at q + j for all j < k (0: d does not hold the phrase)
__device__ uint32_t phrase_match_count(const DevIndex &ix, const DevStep *args, uint32_t k, uint32_t d) {
        const PhraseTerm t0 = phrase_term(ix, phrase_arg(args, 0));
        const HitsView   hv = hits_view(ix);
        HitCursor        c0 = hit_cursor(hv, t0, d);
        uint32_t         total = 0;
        while (c0.left) { // chunks of 64 positions of t0
                const uint32_t     nchunk = min(64u, c0.left);
                unsigned long long alive  = nchunk == 64u ? ~0ull : ((1ull << nchunk) - 1ull);
                for (uint32_t j = 1; j < k && alive; ++j) {
                        const uint32_t tj = phrase_arg(args, j);
                        HitCursor      a  = c0;
                        HitCursor      b;
                        if (tj == 0xffffffffu) {
                                b.p    = nullptr;
                                b.left = b.pos = b.psize = b.mode = 0;
                        } else
                                b = hit_cursor(hv, phrase_term(ix, tj), d);
                        unsigned long long ok = 0;
                        uint32_t           pb = 0;
                        bool               have = false;
                        for (uint32_t r = 0; r < nchunk; ++r) {
                                const uint32_t pa = a.next();
                                if (j == 1u && pa == 0u)
                                        alive &= ~(1ull << r); // position 0 never starts a phrase (docset_iterators.cpp:107)
                                const uint32_t target = pa + j;
                                while ((!have || pb < target) && b.left) { // t(j)'s smallest position >= target (both streams ascend)
                                        pb   = b.next();
                                        have = true;
                                }
                                if (have && pb == target)
                                        ok |= 1ull << r;
                        }
                        alive &= ok;
                }
                total += uint32_t(__popcll(alive));
                for (uint32_t r = 0; r < nchunk; ++r) // t0's cursor moves behind the chunk
                        (void)c0.next();
        }
        return total;
}

// the position filter over the candidates of slot `slot` (NW words, docIDs lo + 32 w + bit); every thread of `nthreads` owns whole words
__device__ void phrase_check(const DevIndex &ix, const DevStep *args, uint32_t k, uint32_t lo, uint32_t NW, uint32_t *slot, float *acc, double idf, int tid, int nthreads) {
        for (uint32_t wi = uint32_t(tid); wi < NW; wi += uint32_t(nthreads)) {
                uint32_t w = slot[wi], keep = w;
                while (w) {
                        const uint32_t bit = uint32_t(__ffs(int(w)) - 1);
                        w &= w - 1;
                        const uint32_t rel = wi * 32u + bit;
                        const uint32_t cnt = phrase_match_count(ix, args, k, lo + rel);
                        if (!cnt)
                                keep &= ~(1u << bit);
                        else if (acc)
                                acc[rel] += bm25_score(idf, cnt);
                }
                slot[wi] = keep;
        }
}
