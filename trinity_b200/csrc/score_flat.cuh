// k_score_flat — scored FLAT disjunctions (a k-term OR or a single term: the ENT::matchanyterms run under AccumulatedScoreScheme) on the
// LUCENE codec: the 10-term OR / BM25 / top-100 workload.  (Included by kernels.cu.)
//
// Replaces (reference): DocsSetSpanForDisjunctionsWithThreshold::process (docset_spans.cpp:681-790: 8192-document window, tracker[] score
// sums), DisjunctionAllPLI next/advance (docset_iterators.cpp:350-405), Lucene refill_documents + FastPFor<4> __decodeArray
// (lucene_codec.cpp:515-594, fastpfor.h:222-270), Scorer::score (similarity.h:228-235) and the application's top-k sink (matches.h:155-171).
//
// Why a second scored kernel: the general step-program kernel (k_exec_tiles) runs a disjunction term after term with a CTA barrier in
// between — on this workload it spends several warp-instructions per posting, with low issue utilisation and
// warps stalled on barriers: half of the ten terms of a query have at most one block in a tile, and three of four warps
// wait while one decodes it.  Here
//   * a tile's blocks of ALL terms form one flat (term, block) list that the 8 warps consume round-robin, with NO barrier between terms:
//     scores are added to the fp32 tile with shared-memory atomics (a document can be hit by two warps working on different terms);
//   * a block's bytes arrive by ONE 1-D bulk copy (cp.async.bulk + mbarrier, issued by one lane, double-buffered per warp) instead of
//     a register-staged copy loop;
//   * a PFor page is unpacked "vertically" (lane l owns values l, l+32, l+64, l+96: one bit position for all four groups), so the
//     consecutive lanes of a warp hit consecutive documents (few bank conflicts in the score tile);
//   * the score tile starts at -0.0f: BM25 contributions are >= +0.0, x + (-0.0) == x, and a document matched iff its word is no
//     longer the sentinel — a flat disjunction needs no docset bitmap at all;
//   * the per-term 64-entry BM25 table is computed once per batch (k_build_luts), not once per (tile, term);
//   * a block that straddles a tile boundary (every block of a sparse term does) is decoded ONCE per run: its documents and scores stay in a
//     per-leaf shared-memory cache and the following tiles just apply them;
//   * top-k: a work item is a RUN of consecutive tiles of one query whose candidate list and threshold live in shared memory across the
//     run; items are handed out run-major (every query's first run, then every query's second run, ...), so when a query's later runs
//     start its first run has already published a threshold — only ~1 in nruns tiles sees the expensive "everything passes" start.
#pragma once

static constexpr uint32_t kSfMaxLeaves = 16;
static constexpr uint32_t kSfStage     = 2080;  // one Lucene block: two int-blocks of at most 1 + 4*255 bytes, + 15 bytes of skew, 16 B multiple
static constexpr uint32_t kSfScratch   = 512;   // 128 words: exception patches of one int-block
static constexpr uint32_t kSfWarpBytes = 2 * kSfStage + kSfScratch;
static constexpr uint32_t kSfSentinel  = 0x80000000u; // -0.0f

// ---- mbarrier + 1-D bulk copy (TMA engine; SASS: UBLKCP / SYNCS)
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
                     : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
        asm volatile("{\n"
                     ".reg .pred P1;\n"
                     "LAB_WAIT:\n"
                     "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
                     "@P1 bra DONE;\n"
                     "bra LAB_WAIT;\n"
                     "DONE:\n"
                     "}" ::"r"(bar),
                     "r"(parity)
                     : "memory");
}

// One int-block (lucene_codec.cpp:69-100 + FastPFor<4> page, fastpfor.h:222-270; SURVEY.md Appendix A) decoded by one warp, lane l
// receiving values l, l+32, l+64, l+96 (v[g] = value l + 32 g).  `s` = 16 B-aligned shared staging, `o` = byte offset of the u8 L.
// Returns the byte offset just past the int-block.
// `bits`: an upper bound of the values' width (b, or maxbits when the page holds exceptions).
__device__ __forceinline__ uint32_t lucene_intblock_v(const uint8_t *s, uint32_t o, int lane, uint32_t v[4], uint32_t *scratch /*128 words, warp-private*/, uint32_t &bits) {
        const uint32_t L = s[o];
        if (L == 0) { // all 128 values equal
                const uint8_t *p = s + o + 1;
                const uint32_t x = varbyte_get(p);
                v[0] = v[1] = v[2] = v[3] = x;
                bits                      = 32u - uint32_t(__clz(int(x)));
                return uint32_t(p - s);
        }
        const uint32_t pw        = o + 1; // byte offset of page word 0 (unaligned)
        const uint32_t wheremeta = lds_u32_unaligned(s, pw + 4);
        const uint32_t b         = (wheremeta - 1u) >> 2;
        v[0] = v[1] = v[2] = v[3] = 0;
        if (b) {
                // group g occupies b words from page word 2 + g*b; value j of a group sits at bit j*b: the same bit position for all four groups.
                // The value's first bit is bit (bit0 & 31) of the aligned shared-memory word that holds it — the page's byte misalignment
                // (0..3 bytes) and the value's bit offset fold into ONE funnel shift of at most 31 over two aligned words (a value has <= 32 bits)
                const uint32_t bit0 = (pw + 8u) * 8u + uint32_t(lane) * b, sh = bit0 & 31u;
                const uint32_t mask = b >= 32u ? 0xffffffffu : ((1u << b) - 1u);
                const uint32_t *w   = reinterpret_cast<const uint32_t *>(s) + (bit0 >> 5);
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                        const uint32_t *wg = w + g * b;
                        v[g]               = __funnelshift_r(wg[0], wg[1], sh) & mask;
                }
        }
        const uint32_t meta     = pw + (1u + wheremeta) * 4u; // byte offset of the bytesize word
        const uint32_t bytesize = lds_u32_unaligned(s, meta);
        const uint8_t *bytes    = s + meta + 4;
        const uint32_t cexcept  = bytes[1];
        bits                    = b;
        if (cexcept) {
                bits = bytes[2];
                // out[pos] |= exc << b (fastpfor.h:248-266); exception e belongs to lane e, the patches travel through the scratch
                const uint32_t maxbits = bytes[2];
                const uint32_t k       = maxbits - b;
                const uint32_t excw    = meta + 4u + ((bytesize + 3u) & ~3u) + 8u; // past the bitmap word and the count word
#pragma unroll
                for (int g = 0; g < 4; ++g)
                        scratch[lane + 32 * g] = 0;
                __syncwarp();
                for (uint32_t e = uint32_t(lane); e < cexcept; e += 32u) {
                        const uint32_t pos = bytes[3 + e] & 127u;
                        uint32_t       ev  = 1;
                        if (k > 1u) {
                                const uint32_t ebp = e * k, wi = ebp >> 5, esh = ebp & 31u;
                                uint32_t       x   = lds_u32_unaligned(s, excw + wi * 4u) >> esh;
                                if (esh + k > 32u)
                                        x |= lds_u32_unaligned(s, excw + wi * 4u + 4u) << (32u - esh);
                                ev = k >= 32u ? x : (x & ((1u << k) - 1u));
                        }
                        scratch[pos] = b >= 32u ? 0u : (ev << b); // positions are distinct within a block
                }
                __syncwarp();
#pragma unroll
                for (int g = 0; g < 4; ++g)
                        v[g] |= scratch[lane + 32 * g];
                __syncwarp();
        }
        return pw + L * 4u;
}

// acc[rel[g]] += sc[g] for the postings selected by `on` (bit g), atomically (another warp may be adding another term's score to the
// same document).  Shared memory has no native fp32 add: atomicAdd compiles to a load / add / compare-and-swap loop per posting, and four
// of them in a row are four serialised ~100-cycle chains.  Here the four loads, adds and CAS attempts are issued side by side; a CAS that
// lost a race (rare) retries on its own.  (Measured alternative: scores as u32 fixed-point units with native ATOMS.ADD — same instruction count, the
// uncontended CAS chains cost little, and slower on the 10-term OR workload; not kept.)
__device__ __forceinline__ void sf_add4(float *acc, const uint32_t rel[4], const float sc[4], uint32_t on) {
        uint32_t *a = reinterpret_cast<uint32_t *>(acc);
        uint32_t  old[4], seen[4];
#pragma unroll
        for (int g = 0; g < 4; ++g)
                old[g] = ((on >> g) & 1u) ? a[rel[g]] : 0u;
#pragma unroll
        for (int g = 0; g < 4; ++g)
                seen[g] = ((on >> g) & 1u) ? atomicCAS(&a[rel[g]], old[g], __float_as_uint(__uint_as_float(old[g]) + sc[g])) : old[g];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
                uint32_t o = old[g], r = seen[g];
                while (r != o) { // lost a race: retry from the value the CAS saw
                        o = r;
                        r = atomicCAS(&a[rel[g]], o, __float_as_uint(__uint_as_float(o) + sc[g]));
                }
        }
}

// per-term BM25 table: lut[leaf][f] = Scorer::score(f) for f < 64 (similarity.h:228-235), once per batch
__global__ void __launch_bounds__(256) k_build_luts(const FlatLeaf *leaves, uint32_t nleaves, float *luts) {
        const uint32_t i = blockIdx.x * 256u + threadIdx.x;
        if (i < nleaves * 64u)
                luts[i] = bm25_score(leaves[i >> 6].idf, i & 63u);
}

// descending prune of the run's candidate list to its k best (list sorted afterwards); returns the new score-bits threshold.
// Called by ALL threads; *s_n is read after a barrier the caller has passed.
// candidate keys kept per run: a power of two (the prune sorts in place) >= kMaxK + 4 * threads (a scan round adds at most 4 keys per thread)
template <int NT> struct SfCap {
        static constexpr uint32_t value = NT <= 384 ? 2048u : 4096u;
};
template <int NT> __device__ __forceinline__ uint32_t sf_prune(unsigned long long *list, uint32_t *s_n, uint32_t k) {
        const uint32_t n  = min(*s_n, SfCap<NT>::value);
        const uint32_t n2 = next_pow2(max(n, 2u));
        __syncthreads();
        for (uint32_t i = n + threadIdx.x; i < n2; i += NT)
                list[i] = 0ull;
        __syncthreads();
        cta_bitonic_desc(list, n2);
        const uint32_t kept = min(n, k);
        const uint32_t thr  = kept == k ? uint32_t(list[k - 1] >> 32) : 0u;
        __syncthreads();
        if (threadIdx.x == 0)
                *s_n = kept;
        __syncthreads();
        return thr;
}

static constexpr uint32_t kSfCacheLeaves = 12;                        // leaves that own a cache slot (the others always decode)
static constexpr uint32_t kSfCacheBytes  = kSfCacheLeaves * 128 * 8;  // per leaf: 128 docIDs + 128 scores of its cached (tile-straddling) block

// FILT: the instantiation for batches that hold a query with a document filter (ScoreParams::filters)
template <int NT, bool FILT>
__global__ void __launch_bounds__(NT, NT <= 384 ? 2 : 1) k_score_flat(ScoreParams S) {
        constexpr int      NWARPS       = NT / 32;
        constexpr uint32_t kSfListCap   = SfCap<NT>::value;
        constexpr uint32_t kSfListBytes = kSfListCap * 8;
        static_assert(kSfListCap >= kMaxK + 4 * NT, "a scan round must fit behind the k best");
        const uint32_t W = 1u << S.tile_shift, W4 = W >> 2, NW = W >> 5;
        float *             acc   = reinterpret_cast<float *>(dyn_smem);
        unsigned long long *list  = reinterpret_cast<unsigned long long *>(dyn_smem + size_t(W) * 4);               // top-k: candidate keys
        uint32_t *          bmap  = reinterpret_cast<uint32_t *>(list);                                           // scored-all: match bitmap (NW words)
        float *             lut   = reinterpret_cast<float *>(dyn_smem + size_t(W) * 4 + kSfListBytes);            // kSfMaxLeaves x 64
        uint32_t *          cdoc  = reinterpret_cast<uint32_t *>(dyn_smem + size_t(W) * 4 + kSfListBytes + size_t(kSfMaxLeaves) * 256); // [leaf][128]
        float *             csc   = reinterpret_cast<float *>(cdoc + kSfCacheLeaves * 128);                        // [leaf][128]
        uint8_t *           wst   = reinterpret_cast<uint8_t *>(csc + kSfCacheLeaves * 128);                       // NWARPS x kSfWarpBytes

        __shared__ __align__(8) unsigned long long s_bar[NWARPS * 2];
        __shared__ uint32_t           s_item, s_n, s_theta, s_warp[NWARPS + 1];
        __shared__ uint32_t           s_fill_blk[2][kSfMaxLeaves], s_fill_tile[2][kSfMaxLeaves]; // block cached for a leaf during tile T: slot T & 1
        __shared__ unsigned long long s_base;

        const int      tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
        uint8_t *      stage   = wst + size_t(warp) * kSfWarpBytes;
        uint32_t *     scratch = reinterpret_cast<uint32_t *>(stage + 2 * kSfStage);
        const uint32_t stage_s = uint32_t(__cvta_generic_to_shared(stage));
        const uint32_t bar_s   = uint32_t(__cvta_generic_to_shared(&s_bar[warp * 2]));
        if (lane == 0) {
                mbar_init(bar_s, 1);
                mbar_init(bar_s + 8, 1);
                asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        uint32_t seq_issue = 0, seq_wait = 0; // bulk copies issued / consumed by this warp: buffer = seq & 1, phase parity = (seq >> 1) & 1
        const float4 sent4 = make_float4(__uint_as_float(kSfSentinel), __uint_as_float(kSfSentinel), __uint_as_float(kSfSentinel), __uint_as_float(kSfSentinel));

        for (;;) {
                __syncthreads();
                if (tid == 0)
                        s_item = atomicAdd(S.ticket, 1u);
                __syncthreads();
                const uint32_t item = s_item;
                if (item >= S.total_items)
                        break;
                // ---- locate the work item
                uint32_t f, run = 0;
                if (S.mode == 2) { // run-major: item = run * nflat + query
                        run = item / S.nflat;
                        f   = item - run * S.nflat;
                } else { // query-major (query, tile) items
                        uint32_t a = 0, b = S.nflat;
                        while (b - a > 1) {
                                const uint32_t mid = (a + b) >> 1;
                                if (S.fq[mid].local_base <= item) a = mid;
                                else b = mid;
                        }
                        f = a;
                }
                const FlatQuery FQ = S.fq[f];
                uint32_t        t0, t1;
                if (S.mode == 2) {
                        if (run >= FQ.nruns)
                                continue;
                        t0 = FQ.tile_lo + run * S.run_tiles;
                        t1 = min(FQ.tile_lo + FQ.ntiles, t0 + S.run_tiles);
                } else {
                        t0 = FQ.tile_lo + (item - FQ.local_base);
                        t1 = t0 + 1u;
                }
                const uint32_t q = FQ.qid, nleaf = FQ.nleaf, k = S.k;
                // ---- lane t adopts leaf t
                uint32_t mydir = 0, mynb = 0, mydocs = 0, myfirst = 0, mylast = 0, mytfb = 0, mytfbase = 0, mytfs = 32;
                double   myidf = 0.0;
                if (uint32_t(lane) < nleaf) {
                        const FlatLeaf Lf = S.leaves[FQ.leaf_begin + lane];
                        myidf             = Lf.idf;
                        if (Lf.term != kEmptyTerm) {
                                const DevTerm T = S.ix.terms[Lf.term];
                                mydir           = T.dir_begin;
                                mynb            = T.nblocks;
                                mydocs          = T.documents;
                                myfirst         = T.first_doc;
                                mylast          = T.last_doc;
                                mytfb           = T.tf_begin;
                                mytfbase        = T.tf_base;
                                mytfs           = T.tf_shift;
                        }
                }
                for (uint32_t i = tid; i < nleaf * 64u; i += NT)
                        lut[i] = S.luts[size_t(FQ.leaf_begin) * 64u + i];
                for (uint32_t i = tid; i < W4; i += NT)
                        reinterpret_cast<float4 *>(acc)[i] = sent4;
                if (tid < 2 * int(kSfMaxLeaves))
                        (&s_fill_tile[0][0])[tid] = 0xffffffffu;
                if (tid == 0)
                        s_n = 0;
                uint32_t thr_local = 0, nmatch = 0, n_list = 0; // n_list: s_n as of the last point where nobody was pushing (same in every thread)
                uint32_t mycb = 0xffffffffu;                    // lane t: the block of leaf t whose documents + scores sit in the cache (same in every warp)
                // first block of every leaf that can reach the run's first document; afterwards each tile's end lookup is the next tile's start
                uint32_t nextA = mynb ? first_block_ge(S.ix, mydir, mynb, myfirst, mylast, mytfb, mytfbase, mytfs, t0 << S.tile_shift) : 0u;
                __syncthreads();

                for (uint32_t tile = t0; tile < t1; ++tile) {
                        const uint32_t lo = tile << S.tile_shift, hi = lo + W; // hi wraps to 0 for the last tile of a 2^32 docID space
                        const uint32_t par = tile & 1u;
                        if (S.mode == 2 && tid == 0)
                                s_theta = *reinterpret_cast<volatile uint32_t *>(&S.theta[q]);
                        // a block cached during the previous tile (by whichever warp decoded it) becomes this leaf's cached block
                        if (uint32_t(lane) < nleaf && tile != t0 && s_fill_tile[par ^ 1u][lane] == tile - 1u)
                                mycb = s_fill_blk[par ^ 1u][lane];
                        // ---- the tile's blocks of every leaf
                        uint32_t bA = nextA, cnt = 0;
                        if (mynb && bA < mynb) {
                                const uint32_t e = (hi == 0u || hi > mylast) ? mynb : first_block_ge(S.ix, mydir, mynb, myfirst, mylast, mytfb, mytfbase, mytfs, hi);
                                nextA            = e;
                                const uint32_t prevLast = bA ? __ldg(S.ix.blk_last + mydir + bA - 1u) : 0u; // documents of block bA start after this
                                if (prevLast + 1u < hi || hi == 0u)
                                        cnt = min(e, mynb - 1u) - bA + 1u;
                                if (lo > mylast)
                                        cnt = 0;
                        }
                        const bool usesCache = cnt && bA == mycb; // the leaf's first block of this tile is the cached one: applied, not decoded
                        if (!usesCache && !(cnt && nextA == mycb))
                                mycb = 0xffffffffu;                  // the cached block ends before the next tile: forget it
                        const uint32_t incl  = warp_incl_scan(cnt, lane);
                        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
                        // ---- this warp's (term, block) pairs: p = warp + NWARPS * j
                        for (uint32_t jb = 0;; jb += 32u) {
                                const uint32_t p    = uint32_t(warp) + NWARPS * (jb + uint32_t(lane));
                                const bool     have = p < total;
                                const uint32_t hm   = __ballot_sync(0xffffffffu, have);
                                if (!hm)
                                        break;
                                uint32_t t = 0;
                                for (uint32_t kk = 0; kk + 1u < nleaf; ++kk)
                                        t += (p >= __shfl_sync(0xffffffffu, incl, int(kk))) ? 1u : 0u;
                                if (!have)
                                        t = 0;
                                const uint32_t tincl = __shfl_sync(0xffffffffu, incl, int(t)), tcnt = __shfl_sync(0xffffffffu, cnt, int(t));
                                const uint32_t tbA   = __shfl_sync(0xffffffffu, bA, int(t));
                                const uint32_t b     = tbA + (p - (tincl - tcnt));
                                const uint32_t dir   = __shfl_sync(0xffffffffu, mydir, int(t));
                                const uint32_t docs  = __shfl_sync(0xffffffffu, mydocs, int(t));
                                const bool     tuse  = __shfl_sync(0xffffffffu, usesCache ? 1 : 0, int(t)) != 0;
                                // kind: 0 = decode, 1 = apply the leaf's cached block, 2 = decode and cache (the leaf's last block of the tile, if the leaf
                                // does not read its cache in this tile: a straddling block will be this leaf's first block of the next tile)
                                uint32_t kind = 0;
                                if (have) {
                                        if (tuse && b == tbA)
                                                kind = 1;
                                        else if (!tuse && b == tbA + tcnt - 1u && b < (docs >> 7) && t < kSfCacheLeaves)
                                                kind = 2;
                                }
                                uint32_t off = 0, offn = 0, prev = 0;
                                if (have && kind != 1u) {
                                        off  = __ldg(S.ix.blk_off + dir + b);
                                        offn = __ldg(S.ix.blk_off + dir + b + 1u);
                                        prev = b ? __ldg(S.ix.blk_last + dir + b - 1u) : 0u;
                                }
                                const uint32_t npairs = __popc(hm);
                                auto issue = [&](uint32_t j) { // bulk copy of pair j's block (cached pairs need no bytes)
                                        if (__shfl_sync(0xffffffffu, kind, int(j)) == 1u)
                                                return;
                                        const uint32_t o = __shfl_sync(0xffffffffu, off, int(j)), on = __shfl_sync(0xffffffffu, offn, int(j));
                                        const uint32_t abase = o & ~15u, bytes = min(((on + 15u) & ~15u) - abase, kSfStage);
                                        if (lane == 0) {
                                                const uint32_t bsel = seq_issue & 1u;
                                                mbar_expect_tx(bar_s + bsel * 8u, bytes);
                                                bulk_g2s(stage_s + bsel * kSfStage, S.ix.index + abase, bytes, bar_s + bsel * 8u);
                                        }
                                        ++seq_issue;
                                };
                                issue(0);
                                for (uint32_t j = 0; j < npairs; ++j) {
                                        if (j + 1u < npairs)
                                                issue(j + 1u);
                                        const uint32_t kj = __shfl_sync(0xffffffffu, kind, int(j));
                                        const uint32_t tj = __shfl_sync(0xffffffffu, t, int(j));
                                        const float *  lt = lut + tj * 64u;
                                        if (kj == 1u) {
                                                // ---- cached block: its documents and scores were left behind by an earlier tile of this run
                                                uint32_t rel[4], on = 0;
                                                float    sc[4];
#pragma unroll
                                                for (int g = 0; g < 4; ++g) {
                                                        rel[g] = cdoc[tj * 128u + lane + 32 * g] - lo;
                                                        sc[g]  = csc[tj * 128u + lane + 32 * g];
                                                        on |= (rel[g] < W ? 1u : 0u) << g;
                                                }
                                                sf_add4(acc, rel, sc, on);
                                                continue;
                                        }
                                        const uint32_t bsel = seq_wait & 1u;
                                        mbar_wait(bar_s + bsel * 8u, (seq_wait >> 1) & 1u);
                                        ++seq_wait;
                                        const uint8_t *s    = stage + bsel * kSfStage;
                                        const uint32_t oj   = __shfl_sync(0xffffffffu, off, int(j));
                                        const uint32_t bj   = __shfl_sync(0xffffffffu, b, int(j));
                                        const uint32_t pj   = __shfl_sync(0xffffffffu, prev, int(j));
                                        const uint32_t dj   = __shfl_sync(0xffffffffu, docs, int(j));
                                        const uint32_t skew = oj & 15u;
                                        if (bj < (dj >> 7)) {
                                                uint32_t d[4], fr[4], dbits, fbits;
                                                const uint32_t o2 = lucene_intblock_v(s, skew, lane, d, scratch, dbits);
                                                (void)lucene_intblock_v(s, o2, lane, fr, scratch, fbits);
                                                // docIDs = prev + inclusive prefix sum over the block (lucene_codec.cpp:568-594 update_curdoc), group by group
                                                uint32_t last;
                                                if (dbits <= 11u) { // 32 values below 2048 sum to less than 65536: two groups share one scan
                                                        const uint32_t sa = warp_incl_scan(d[0] | (d[1] << 16), lane), sb = warp_incl_scan(d[2] | (d[3] << 16), lane);
                                                        const uint32_t ta = __shfl_sync(0xffffffffu, sa, 31), tb = __shfl_sync(0xffffffffu, sb, 31);
                                                        const uint32_t b1 = pj + (ta & 0xffffu), b2 = b1 + (ta >> 16), b3 = b2 + (tb & 0xffffu);
                                                        d[0] = pj + (sa & 0xffffu);
                                                        d[1] = b1 + (sa >> 16);
                                                        d[2] = b2 + (sb & 0xffffu);
                                                        d[3] = b3 + (sb >> 16);
                                                        last = b3 + (tb >> 16);
                                                } else {
                                                        uint32_t base = pj;
#pragma unroll
                                                        for (int g = 0; g < 4; ++g) {
                                                                const uint32_t sc = warp_incl_scan(d[g], lane);
                                                                d[g]              = base + sc;
                                                                base += __shfl_sync(0xffffffffu, sc, 31);
                                                        }
                                                        last = base;
                                                }
                                                const bool big = fbits > 6u; // some freq may be >= 64: outside the table
                                                double     idfj = 0.0;
                                                if (big)
                                                        idfj = __shfl_sync(0xffffffffu, myidf, int(tj));
                                                const uint32_t first = __shfl_sync(0xffffffffu, d[0], 0);
                                                // the four scores (table look-ups side by side) and tile-relative documents of this lane
                                                float    sc[4];
                                                uint32_t rel[4], on = 0;
#pragma unroll
                                                for (int g = 0; g < 4; ++g) {
                                                        const uint32_t f16 = fr[g] & 0xffffu; // freq is uint16_t in the reference (codecs.h:217)
                                                        sc[g]              = (!big || f16 < 64u) ? lt[f16 & 63u] : bm25_score(idfj, f16);
                                                        rel[g]             = d[g] - lo;
                                                }
                                                if (first - lo < W && last - lo < W)
                                                        on = 0xfu; // block completely inside the tile: no range checks
                                                else {
#pragma unroll
                                                        for (int g = 0; g < 4; ++g)
                                                                on |= (rel[g] < W ? 1u : 0u) << g;
                                                }
                                                sf_add4(acc, rel, sc, on);
                                                if (kj == 2u) { // the leaf's last block of the tile: keep it for the following tiles of the run
#pragma unroll
                                                        for (int g = 0; g < 4; ++g) {
                                                                cdoc[tj * 128u + lane + 32 * g] = d[g];
                                                                csc[tj * 128u + lane + 32 * g]  = sc[g];
                                                        }
                                                        if (lane == 0 && (hi != 0u && last >= hi)) { // it does reach into the next tile
                                                                s_fill_blk[par][tj]  = bj;
                                                                s_fill_tile[par][tj] = tile;
                                                        }
                                                }
                                        } else {
                                                // tail block: (varbyte delta, varbyte freq) pairs (lucene_codec.cpp:527-550)
                                                const double idfj = __shfl_sync(0xffffffffu, myidf, int(tj));
                                                if (lane == 0) {
                                                        const uint8_t *pp   = s + skew;
                                                        const uint32_t tail = dj & 127u;
                                                        uint32_t       doc  = pj;
                                                        for (uint32_t i = 0; i < tail; ++i) {
                                                                doc += varbyte_get(pp);
                                                                const uint32_t f16 = varbyte_get(pp) & 0xffffu;
                                                                const uint32_t rel = doc - lo;
                                                                if (rel < W)
                                                                        atomicAdd(&acc[rel], f16 < 64u ? lt[f16] : bm25_score(idfj, f16));
                                                        }
                                                }
                                        }
                                        __syncwarp();
                                }
                        }
                        __syncthreads(); // ---- every posting of the tile has been scored

                        if constexpr (FILT) { // the documents the query's filter drops leave the score tile: not counted, no candidate slot, no theta
                                const DevFilter F = S.filters[q];
                                for (uint32_t i4 = tid; i4 < W4; i4 += NT) {
                                        const uint32_t m = (filter_keep(F, (lo >> 5) + (i4 >> 3)) >> ((i4 & 7u) * 4u)) & 0xfu;
                                        if (m != 0xfu) {
                                                float4 v = reinterpret_cast<const float4 *>(acc)[i4];
                                                if (!(m & 1u)) v.x = sent4.x;
                                                if (!(m & 2u)) v.y = sent4.y;
                                                if (!(m & 4u)) v.z = sent4.z;
                                                if (!(m & 8u)) v.w = sent4.w;
                                                reinterpret_cast<float4 *>(acc)[i4] = v;
                                        }
                                }
                                __syncthreads();
                        }

                        const uint32_t *mk = S.ix.masked ? S.ix.masked + (lo >> 5) : nullptr;
                        if (S.mode == 2) {
                                // ---- threshold scan: as signed integers the sentinel is INT_MIN and scores (>= +0.0) order like their bits
                                const int      thr      = int(max(thr_local, s_theta));
                                const uint32_t n_before = n_list;
                                for (uint32_t i4 = tid; i4 < W4; i4 += NT) {
                                        float4   v  = reinterpret_cast<const float4 *>(acc)[i4];
                                        uint32_t b0 = __float_as_uint(v.x), b1 = __float_as_uint(v.y), b2 = __float_as_uint(v.z), b3 = __float_as_uint(v.w);
                                        if (mk) { // masked documents (masked_documents_registry::test, exec.cpp:1108-1116) never reach the sink
                                                const uint32_t m = (__ldg(mk + (i4 >> 3)) >> ((i4 & 7u) * 4u)) & 0xfu;
                                                if (m & 1u) b0 = kSfSentinel;
                                                if (m & 2u) b1 = kSfSentinel;
                                                if (m & 4u) b2 = kSfSentinel;
                                                if (m & 8u) b3 = kSfSentinel;
                                        }
                                        nmatch += 4u - ((b0 >> 31) + (b1 >> 31) + (b2 >> 31) + (b3 >> 31));
                                        if (max(max(int(b0), int(b1)), max(int(b2), int(b3))) >= thr) {
                                                const uint32_t bb[4] = {b0, b1, b2, b3};
#pragma unroll
                                                for (int c = 0; c < 4; ++c)
                                                        if (int(bb[c]) >= thr) {
                                                                const uint32_t idx = atomicAdd(&s_n, 1u);
                                                                if (idx < kSfListCap)
                                                                        list[idx] = (static_cast<unsigned long long>(bb[c]) << 32) | static_cast<unsigned long long>(~(lo + i4 * 4u + c));
                                                        }
                                        }
                                }
                                __syncthreads();
                                if (s_n > kSfListCap) {
                                        // more candidates than the list holds (only while the threshold is still ~0): redo the tile in rounds of
                                        // NT * 4 documents, pruning to the k best whenever the next round might not fit
                                        __syncthreads();
                                        if (tid == 0)
                                                s_n = n_before;
                                        __syncthreads();
                                        for (uint32_t r4 = 0; r4 < W4; r4 += NT) {
                                                __syncthreads();
                                                const uint32_t cur = s_n; // read between two barriers: nobody is pushing
                                                __syncthreads();
                                                if (cur + 4u * NT > kSfListCap)
                                                        thr_local = max(thr_local, sf_prune<NT>(list, &s_n, k));
                                                const uint32_t i4 = r4 + tid;
                                                if (i4 < W4) {
                                                        const int thr2 = int(max(thr_local, uint32_t(thr)));
                                                        float4    v    = reinterpret_cast<const float4 *>(acc)[i4];
                                                        uint32_t  bb[4] = {__float_as_uint(v.x), __float_as_uint(v.y), __float_as_uint(v.z), __float_as_uint(v.w)};
                                                        if (mk) {
                                                                const uint32_t m = (__ldg(mk + (i4 >> 3)) >> ((i4 & 7u) * 4u)) & 0xfu;
#pragma unroll
                                                                for (int c = 0; c < 4; ++c)
                                                                        if ((m >> c) & 1u)
                                                                                bb[c] = kSfSentinel;
                                                        }
#pragma unroll
                                                        for (int c = 0; c < 4; ++c)
                                                                if (int(bb[c]) >= thr2) {
                                                                        const uint32_t idx = atomicAdd(&s_n, 1u);
                                                                        list[idx] = (static_cast<unsigned long long>(bb[c]) << 32) | static_cast<unsigned long long>(~(lo + i4 * 4u + c));
                                                                }
                                                }
                                        }
                                        __syncthreads();
                                }
                                if (s_n > kSfListCap / 2u)
                                        thr_local = max(thr_local, sf_prune<NT>(list, &s_n, k));
                        } else {
                                // ---- scored-all: match bitmap out of the score tile, then the ordered compaction of k_exec_tiles
                                for (uint32_t r4 = 0; r4 < W4; r4 += NT) { // (every lane of a warp takes part in the shuffles: W4 is a multiple of 32)
                                        const uint32_t i4  = r4 + tid;
                                        const bool     on  = i4 < W4;
                                        const float4   v   = on ? reinterpret_cast<const float4 *>(acc)[i4] : sent4;
                                        uint32_t       nib = ((~__float_as_uint(v.x)) >> 31) | (((~__float_as_uint(v.y)) >> 31) << 1) | (((~__float_as_uint(v.z)) >> 31) << 2) |
                                                       (((~__float_as_uint(v.w)) >> 31) << 3);
                                        nib <<= (i4 & 7u) * 4u;
                                        nib |= __shfl_xor_sync(0xffffffffu, nib, 1);
                                        nib |= __shfl_xor_sync(0xffffffffu, nib, 2);
                                        nib |= __shfl_xor_sync(0xffffffffu, nib, 4);
                                        if (on && (i4 & 7u) == 0u)
                                                bmap[i4 >> 3] = mk ? (nib & ~__ldg(mk + (i4 >> 3))) : nib;
                                }
                                __syncthreads();
                                const uint32_t wpt = (NW + NT - 1u) / NT; // bitmap words per thread (contiguous: thread order == docID order)
                                uint32_t       c   = 0;
                                for (uint32_t i = 0; i < wpt; ++i)
                                        if (tid * wpt + i < NW)
                                                c += __popc(bmap[tid * wpt + i]);
                                // CTA exclusive scan
                                const uint32_t inclc = warp_incl_scan(c, lane);
                                if (lane == 31)
                                        s_warp[warp] = inclc;
                                __syncthreads();
                                uint32_t wbase = 0, tot = 0;
#pragma unroll
                                for (int w8 = 0; w8 < NWARPS; ++w8) {
                                        const uint32_t x = s_warp[w8];
                                        if (w8 < warp)
                                                wbase += x;
                                        tot += x;
                                }
                                const uint32_t gitem = FQ.item_base + (tile - FQ.tile_lo);
                                if (tid == 0) {
                                        unsigned long long base = 0;
                                        if (tot) {
                                                base = atomicAdd(S.seg_cursor, static_cast<unsigned long long>(tot));
                                                atomicAdd(&S.match_counts[q], static_cast<unsigned long long>(tot));
                                                if (base + tot > S.seg_capacity) {
                                                        *S.overflow = 1;
                                                        base        = ~0ull;
                                                }
                                        }
                                        s_base            = base;
                                        S.item_off[gitem] = base;
                                        S.item_cnt[gitem] = base == ~0ull ? 0u : tot;
                                }
                                __syncthreads();
                                const unsigned long long base = s_base;
                                if (tot && base != ~0ull) {
                                        unsigned long long pos = base + wbase + (inclc - c);
                                        for (uint32_t i = 0; i < wpt; ++i) {
                                                const uint32_t wi = tid * wpt + i;
                                                uint32_t       w  = wi < NW ? bmap[wi] : 0u;
                                                while (w) {
                                                        const uint32_t bit = uint32_t(__ffs(int(w)) - 1);
                                                        w &= w - 1;
                                                        const uint32_t rel = wi * 32u + bit;
                                                        S.seg_docids[pos]  = lo + rel;
                                                        S.seg_scores[pos]  = acc[rel];
                                                        ++pos;
                                                }
                                        }
                                }
                        }
                        __syncthreads();
                        n_list = s_n;
                        for (uint32_t i = tid; i < W4; i += NT) // the next tile starts from an untouched score tile
                                reinterpret_cast<float4 *>(acc)[i] = sent4;
                        __syncthreads();
                }

                if (S.mode == 2) {
                        // ---- end of the run: its k best (those that can still matter) join the query's candidates; its k-th best bounds the query's
                        if (s_n >= k || s_n > kSfListCap / 2u)
                                thr_local = max(thr_local, sf_prune<NT>(list, &s_n, k));
                        const uint32_t n      = s_n;
                        const uint32_t theta0 = *reinterpret_cast<volatile uint32_t *>(&S.theta[q]);
                        for (uint32_t i = tid; i < n; i += NT) {
                                const unsigned long long key = list[i];
                                if (uint32_t(key >> 32) >= theta0) {
                                        const uint32_t pos = atomicAdd(&S.cand_cursor[q], 1u);
                                        if (pos < FQ.cand_cap)
                                                S.cand[size_t(FQ.cand_base) + pos] = make_uint2(uint32_t(key >> 32), ~uint32_t(key));
                                }
                        }
                        if (n >= k && tid == 0)
                                atomicMax(&S.theta[q], thr_local);
                        for (int d = 16; d > 0; d >>= 1)
                                nmatch += __shfl_xor_sync(0xffffffffu, nmatch, d);
                        if (lane == 0 && nmatch)
                                atomicAdd(&S.match_counts[q], static_cast<unsigned long long>(nmatch));
                }
        }
}

size_t score_flat_smem_bytes(uint32_t tile_shift, int threads) {
        const size_t listBytes = (threads <= 384 ? 2048u : 4096u) * 8u;
        return (size_t(1) << tile_shift) * 4 + listBytes + size_t(kSfMaxLeaves) * 256 + kSfCacheBytes + size_t(threads / 32) * kSfWarpBytes;
}

uint32_t score_flat_max_leaves() {
        return kSfMaxLeaves;
}

cudaError_t launch_build_luts(const FlatLeaf *leaves, uint32_t nleaves, float *luts, cudaStream_t stream) {
        if (!nleaves)
                return cudaSuccess;
        k_build_luts<<<(nleaves * 64u + 255u) / 256u, 256, 0, stream>>>(leaves, nleaves, luts);
        return cudaGetLastError();
}

// threads: CTA size (320: two CTAs per SM on 2^13-document tiles; 512: one CTA per SM, for 2^14-document tiles; any other value runs 320)
cudaError_t launch_score_flat(const ScoreParams &S, int threads, int num_sms, cudaStream_t stream) {
        if (threads != 512)
                threads = 320;
        const void *fn = S.filters ? (threads == 512 ? (const void *)k_score_flat<512, true> : (const void *)k_score_flat<320, true>)
                                   : (threads == 512 ? (const void *)k_score_flat<512, false> : (const void *)k_score_flat<320, false>);
        const size_t smem = score_flat_smem_bytes(S.tile_shift, threads);
        cudaError_t  e    = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
        if (e != cudaSuccess)
                return e;
        int per = 0;
        e       = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, fn, threads, smem);
        if (e != cudaSuccess)
                return e;
        if (per <= 0)
                return cudaErrorLaunchOutOfResources;
        const int grid = int(std::min<uint64_t>(uint64_t(num_sms) * per, std::max<uint32_t>(1u, S.total_items)));
        void *    args[] = {(void *)&S};
        return cudaLaunchKernel(fn, dim3(grid), dim3(threads), args, smem, stream);
}
