// sm_90a kernels of the trinity_b200 hot path.
//
//   k_exec_tiles   fused postings-block decode -> docset algebra -> BM25 accumulate -> emit / top-k candidates
//                  one work item = (query, docID tile of 2^tile_shift docs); persistent CTAs pull items from a ticket.
//                  Replaces (reference): Decoder::unpack_block/next/advance (google_codec.cpp:596-934), Lucene
//                  refill_documents + FastPFor __decodeArray (lucene_codec.cpp:515-594, fastpfor.h:222-270),
//                  Conjuction/Disjunction/Filter/Optional next/advance (docset_iterators.cpp:282-677), the IteratorScorer
//                  wrappers (docset_iterators_scorers.cpp:8-242), BM25 score (similarity.h:228-235) and the span drivers
//                  (docset_spans.cpp:98-173,244-290,681-790).  The 8192-doc window of DocsSetSpanForDisjunctions becomes the
//                  CTA's docID tile; tracker[] becomes the smem score tile; matching[] becomes the smem slot bitmaps.
//   k_item_scan / k_gather   order the per-tile result segments by (query, tile) == ascending docID per query,
//                  the order in which the reference calls MatchedIndexDocumentsFilter::consider() (exec.cpp:1215-1335).
//   k_topk_select  per-query exact top-k (score desc, docID asc) over the per-tile candidates.
//   k_topk_merge   merge of per-shard top-k lists after the all-gather (multi-GPU exchange step, SURVEY.md 8e).
#include "device_types.h"
#include "dirlookup.h"
#include "hitcursor.h"
#include "kernels.h"
#include "varbyte.h"
#include <algorithm>
#include <type_traits>
#include <cuda_runtime.h>

namespace trn {

static constexpr int      kThreads    = 128;
static constexpr int      kWarps      = kThreads / 32;
static constexpr uint32_t kStageBytes = 6144; // per-warp staging area for compressed bytes
static constexpr uint32_t kListCap    = 2048; // smem candidate list (entries) of the select / merge kernels
static constexpr uint32_t kTileListCap = 1024; // per-tile candidate list of k_exec_tiles (k <= 512 kept + 512 docs per round)
static constexpr uint32_t kMaxK       = 512;

// ------------------------------------------------------------------------------------------------ small helpers
__device__ __forceinline__ uint4 ld_stream_v4(const void *p) {
        uint4 r;
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
        return r;
}

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane) {
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
                const uint32_t n = __shfl_up_sync(0xffffffffu, v, d);
                if (lane >= d)
                        v += n;
        }
        return v;
}

// unaligned little-endian u32 from a 4B-aligned shared buffer
__device__ __forceinline__ uint32_t lds_u32_unaligned(const uint8_t *base4, uint32_t byteoff) {
        const uint32_t *w  = reinterpret_cast<const uint32_t *>(base4);
        const uint32_t  i  = byteoff >> 2;
        const uint32_t  sh = (byteoff & 3u) * 8u;
        return __funnelshift_r(w[i], w[i + 1], sh);
}

// Warp-cooperative copy of index bytes [off, off+len) into the warp's staging area; returns the staging byte offset
// that corresponds to `off` (0..15).  16B-aligned 128-bit streaming loads, fully coalesced.
__device__ __forceinline__ uint32_t stage_copy(const uint8_t *__restrict__ index, uint32_t off, uint32_t len, uint8_t *stage, int lane) {
        const uint32_t abase = off & ~15u;
        const uint32_t total = ((off + len + 15u) & ~15u) - abase; // bytes, multiple of 16
        for (uint32_t i = lane * 16u; i < total; i += 512u)
                *reinterpret_cast<uint4 *>(stage + i) = ld_stream_v4(index + abase + i);
        return off - abase;
}

// docID -> block lookup (dirlookup.h) over the device copy of the directory
__device__ __forceinline__ uint32_t first_block_ge(const DevIndex &ix, uint32_t dir_begin, uint32_t nblocks, uint32_t first_doc, uint32_t last_doc, uint32_t tf_begin,
                                                   uint32_t tf_base, uint32_t tf_shift, uint32_t d) {
        return dir_first_block_ge(ix.blk_last + dir_begin, ix.tile_first + tf_begin, nblocks, first_doc, last_doc, tf_base, tf_shift, d);
}
__device__ __forceinline__ uint32_t first_block_ge(const DevIndex &ix, const DevTerm &T, uint32_t d) {
        return first_block_ge(ix, T.dir_begin, T.nblocks, T.first_doc, T.last_doc, T.tf_begin, T.tf_base, T.tf_shift, d);
}
// blocks [bA, bB] of term T that can hold a document of [lo, lo + W): bA > bB when there is none
__device__ __forceinline__ void tile_block_range(const DevIndex &ix, const DevTerm &T, uint32_t lo, uint32_t W, uint32_t &bA, uint32_t &bB) {
        bA = 1u;
        bB = 0u;
        if (!T.nblocks || lo > T.last_doc || lo + (W - 1u) < T.first_doc)
                return;
        const uint32_t a = first_block_ge(ix, T, lo);
        if (a >= T.nblocks)
                return;
        bA = a;
        bB = min(first_block_ge(ix, T, lo + (W - 1u)), T.nblocks - 1u);
}

// BM25 per-posting score == IndexSourcesCollectionBM25Scorer::Scorer::score (similarity.h:228-235)
__device__ __forceinline__ float bm25_score(double idf, uint32_t freq) {
        const float f = float(freq & 0xffffu); // freq is uint16_t in the reference (codecs.h:217, common.h:46)
        return float(idf * double(f) / double(f + 1.2f));
}

// ------------------------------------------------------------------------------------------------ sinks
// Per-lane docset bit builder: consecutive docs of a lane are ascending, so bits are gathered per 32-doc word in a
// register and flushed with ONE shared-memory atomic per word (not per posting).
struct BitSink {
        uint32_t *      bm;   // destination bitmap (shared)
        const uint32_t *filt; // optional filter bitmap: only bits also set here are kept (AND)
        int             mode; // M_OR (or-in), M_ANDNOT (clear), M_NONE
        int             cur_w;
        uint32_t        cur;
        __device__ __forceinline__ void init(uint32_t *b, const uint32_t *f, int m) {
                bm    = b;
                filt  = f;
                mode  = m;
                cur_w = -1;
                cur   = 0;
        }
        __device__ __forceinline__ void flush() {
                if (cur_w >= 0 && cur) {
                        if (mode == M_ANDNOT)
                                atomicAnd(&bm[cur_w], ~cur);
                        else {
                                const uint32_t v = filt ? (cur & filt[cur_w]) : cur;
                                if (v)
                                        atomicOr(&bm[cur_w], v);
                        }
                }
                cur = 0;
        }
        __device__ __forceinline__ void add(uint32_t rel) {
                const int w = int(rel >> 5);
                if (w != cur_w) {
                        flush();
                        cur_w = w;
                }
                cur |= 1u << (rel & 31u);
        }
};

struct LeafCtx {
        uint32_t     lo, hi; // docID range [lo, hi) of the tile
        BitSink      bits;
        bool         want_bits;
        bool         want_score;
        float *      acc;        // shared score tile
        const float *lut;        // shared, 64 entries
        const uint32_t *mask;    // optional: accumulate only where this bitmap has the doc's bit (second pass)
        double       idf;
        __device__ __forceinline__ void visit(uint32_t doc, uint32_t freq) {
                const uint32_t rel = doc - lo;
                if (want_bits)
                        bits.add(rel);
                if (want_score) {
                        if (mask && !((mask[rel >> 5] >> (rel & 31u)) & 1u))
                                return;
                        const uint32_t f16 = freq & 0xffffu;
                        const float s   = f16 < 64u ? lut[f16] : bm25_score(idf, f16);
                        acc[rel] += s; // docs are unique within one term and terms are processed one at a time: no race
                }
        }
};

// ------------------------------------------------------------------------------------------------ GOOGLE block decode
// One lane decodes one 32-doc block (google_codec.cpp:596-639 unpack_block).  p points at the first doc-delta varbyte
// (after the header's n byte).  Layout: (n-1) delta varbytes, n freq varbytes, then hits (never parsed here: the next
// block is found through the directory, not by walking the hits like skip_block_doc google_codec.cpp:497-531).
template <bool NEED_FREQ, class V>
__device__ __forceinline__ void google_block(const uint8_t *p, uint32_t n, uint32_t prev, uint32_t last, uint32_t lo, uint32_t hi, V &v) {
        const uint8_t *pf = p;
        if (NEED_FREQ) {
                for (uint32_t i = 0; i + 1 < n; ++i)
                        pf += varbyte_len(*pf);
        }
        const uint32_t W = hi - lo; // tile membership is doc - lo < W: hi wraps to 0 for the last tile of a 2^32 docID space
        uint32_t       doc = prev;
        for (uint32_t i = 0; i + 1 < n; ++i) {
                doc += varbyte_get(p);
                uint32_t fr = 0;
                if (NEED_FREQ)
                        fr = varbyte_get(pf);
                if (doc >= lo) {
                        if (doc - lo >= W)
                                return;
                        v.visit(doc, fr);
                }
        }
        if (last - lo < W) {
                uint32_t fr = 0;
                if (NEED_FREQ)
                        fr = varbyte_get(pf);
                v.visit(last, fr);
        }
}

// Decode blocks [bA, bB] of term T that overlap the tile; warps take groups of 32 consecutive blocks.
template <bool NEED_FREQ>
__device__ void google_leaf(const DevIndex &ix, const DevTerm &T, uint32_t bA, uint32_t bB, LeafCtx &lc, const uint32_t *skipfilt, uint8_t *stage_all,
                            uint32_t stageBytes) {
        const int       lane  = threadIdx.x & 31, warp = threadIdx.x >> 5;
        uint8_t *       stage = stage_all + warp * stageBytes;
        const uint32_t *bl    = ix.blk_last + T.dir_begin;
        const uint32_t *bo    = ix.blk_off + T.dir_begin;
        for (uint32_t g = bA + warp * 32u; g <= bB; g += kWarps * 32u) {
                const uint32_t b      = g + lane;
                const bool     active = b <= bB;
                uint32_t       off = 0, offn = 0, last = 0, prev = 0, n = 0;
                if (active) {
                        off  = bo[b];
                        offn = bo[b + 1];
                        last = bl[b];
                        prev = b ? bl[b - 1] : 0u;
                        n    = (b + 1 == T.nblocks) ? (T.documents - 32u * (T.nblocks - 1u)) : 32u;
                }
                const uint32_t cnt       = min(32u, bB - g + 1u);
                const uint32_t first_off = __shfl_sync(0xffffffffu, off, 0);
                const uint32_t end_off   = __shfl_sync(0xffffffffu, offn, int(cnt) - 1);
                const uint32_t span      = end_off - first_off;
                // optional block-level skip: the destination docset has no candidate inside this block's docID range
                bool need = active;
                if (need && skipfilt) {
                        const uint32_t d0 = max(prev + 1u, lc.lo), d1 = min(last, lc.hi - 1u);
                        if (d1 < d0)
                                need = false;
                        else {
                                const uint32_t r0 = d0 - lc.lo, r1 = d1 - lc.lo, w0 = r0 >> 5, w1 = r1 >> 5;
                                if (w1 - w0 <= 3u) {
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
                if (span + 32u <= stageBytes) {
                        if (__any_sync(0xffffffffu, need)) {
                                const uint32_t skew = stage_copy(ix.index, first_off, span, stage, lane);
                                __syncwarp();
                                if (need)
                                        google_block<NEED_FREQ>(stage + skew + (off - first_off), n, prev, last, lc.lo, lc.hi, lc);
                        }
                } else if (need) {
                        // hits-heavy blocks that do not fit the staging area: read this block straight from global memory
                        google_block<NEED_FREQ>(ix.index + off, n, prev, last, lc.lo, lc.hi, lc);
                }
                __syncwarp();
        }
        if (lc.want_bits)
                lc.bits.flush();
}

// ------------------------------------------------------------------------------------------------ LUCENE block decode
// One warp decodes one 128-doc block; lane l owns values 4l..4l+3.  int-block format: lucene_codec.cpp:26-100,
// FastPFor<4> page: fastpfor.h:167-270 (see SURVEY.md Appendix A).  `s` = 4B-aligned shared staging, `o` = byte offset of
// the int-block's u8 L.  Returns the byte offset just past the int-block.
__device__ __forceinline__ uint32_t lucene_intblock(const uint8_t *s, uint32_t o, int lane, uint32_t v[4], uint32_t *scratch /*128 words, warp-private*/) {
        const uint32_t L = s[o];
        if (L == 0) {
                const uint8_t *p  = s + o + 1;
                const uint32_t x  = varbyte_get(p);
                v[0] = v[1] = v[2] = v[3] = x;
                return uint32_t(p - s);
        }
        const uint32_t pw        = o + 1; // byte offset of page word 0
        const uint32_t wheremeta = lds_u32_unaligned(s, pw + 4);
        const uint32_t b         = (wheremeta - 1u) >> 2;
        // packed area: words 2 .. 2+4b ; value i (group g = i/32, j = i%32) at bit j*b of group g (b words per group)
        const uint32_t g = uint32_t(lane) >> 3, j0 = (uint32_t(lane) & 7u) * 4u;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
                uint32_t val = 0;
                if (b) {
                        const uint32_t bp = (j0 + t) * b, wi = 2u + g * b + (bp >> 5), sh = bp & 31u;
                        const uint32_t w0 = lds_u32_unaligned(s, pw + wi * 4u);
                        uint32_t       x  = w0 >> sh;
                        if (sh + b > 32u) {
                                const uint32_t w1 = lds_u32_unaligned(s, pw + wi * 4u + 4u);
                                x |= w1 << (32u - sh);
                        }
                        val = b == 32u ? x : (x & ((1u << b) - 1u));
                }
                v[t] = val;
        }
        const uint32_t meta     = pw + (1u + wheremeta) * 4u; // byte offset of bytesize word
        const uint32_t bytesize = lds_u32_unaligned(s, meta);
        const uint8_t *bytes    = s + meta + 4;
        const uint32_t cexcept  = bytes[1];
        if (cexcept) {
                // Exception patching (fastpfor.h:248-266): out[pos] |= exc << b.  Lane e owns exception e; the patched values travel through a
                // warp-private scratch (the first version had EVERY lane walk ALL exceptions: ~15 instructions x cexcept per int-block,
                // the top instruction hot spot of the OR/BM25 workload).
                const uint32_t maxbits = bytes[2];
                const uint32_t k       = maxbits - b;
                const uint32_t excw    = meta + 4u + ((bytesize + 3u) & ~3u) + 8u; // past bitmap word and count word
#pragma unroll
                for (int t = 0; t < 4; ++t)
                        scratch[lane * 4 + t] = v[t];
                __syncwarp();
                for (uint32_t e = uint32_t(lane); e < cexcept; e += 32u) {
                        const uint32_t pos = bytes[3 + e];
                        uint32_t       ev  = 1;
                        if (k > 1u) {
                                const uint32_t bp = e * k, wi = bp >> 5, sh = bp & 31u;
                                uint32_t       x  = lds_u32_unaligned(s, excw + wi * 4u) >> sh;
                                if (sh + k > 32u)
                                        x |= lds_u32_unaligned(s, excw + wi * 4u + 4u) << (32u - sh);
                                ev = k == 32u ? x : (x & ((1u << k) - 1u));
                        }
                        scratch[pos] |= ev << b; // positions are distinct within a block
                }
                __syncwarp();
#pragma unroll
                for (int t = 0; t < 4; ++t)
                        v[t] = scratch[lane * 4 + t];
                __syncwarp();
        }
        return pw + L * 4u;
}

template <bool NEED_FREQ>
__device__ void lucene_leaf(const DevIndex &ix, const DevTerm &T, uint32_t bA, uint32_t bB, LeafCtx &lc, const uint32_t *skipfilt, uint8_t *stage_all,
                            uint32_t stageBytes) {
        const int       lane  = threadIdx.x & 31, warp = threadIdx.x >> 5;
        uint8_t *       stage = stage_all + warp * stageBytes;
        const uint32_t *bl    = ix.blk_last + T.dir_begin;
        const uint32_t *bo    = ix.blk_off + T.dir_begin;
        const uint32_t  nfull = T.documents >> 7;
        for (uint32_t b = bA + warp; b <= bB; b += kWarps) {
                const uint32_t off = bo[b], offn = bo[b + 1], last = bl[b], prev = b ? bl[b - 1] : 0u;
                bool           need = true;
                if (skipfilt) {
                        const uint32_t d0 = max(prev + 1u, lc.lo), d1 = min(last, lc.hi - 1u);
                        if (d1 < d0)
                                need = false;
                        else {
                                const uint32_t r0 = d0 - lc.lo, r1 = d1 - lc.lo, w0 = r0 >> 5, w1 = r1 >> 5;
                                if (w1 - w0 < 32u) { // one filter word per lane
                                        uint32_t m = 0;
                                        const uint32_t w = w0 + lane;
                                        if (w <= w1) {
                                                m = skipfilt[w];
                                                if (w == w0)
                                                        m &= 0xffffffffu << (r0 & 31u);
                                                if (w == w1)
                                                        m &= 0xffffffffu >> (31u - (r1 & 31u));
                                        }
                                        need = __any_sync(0xffffffffu, m != 0);
                                }
                        }
                }
                if (!need)
                        continue;
                const uint32_t len = offn - off;
                if (b < nfull) {
                        // full 128-doc block: two int-blocks (deltas, freqs), at most 2*(1+4*255) bytes
                        const uint32_t skew = stage_copy(ix.index, off, len, stage, lane);
                        __syncwarp();
                        uint32_t d[4], f[4] = {0, 0, 0, 0};
                        const uint32_t o2 = lucene_intblock(stage, skew, lane, d, reinterpret_cast<uint32_t *>(stage + 2560));
                        if (NEED_FREQ)
                                (void)lucene_intblock(stage, o2, lane, f, reinterpret_cast<uint32_t *>(stage + 2560));
                        // docIDs = prev + inclusive prefix sum of deltas (lucene_codec.cpp:568-594 update_curdoc)
                        d[1] += d[0];
                        d[2] += d[1];
                        d[3] += d[2];
                        const uint32_t incl = warp_incl_scan(d[3], lane);
                        const uint32_t base = prev + incl - d[3];
#pragma unroll
                        for (int t = 0; t < 4; ++t) {
                                const uint32_t doc = base + d[t];
                                if (doc - lc.lo < lc.hi - lc.lo) // (not doc < hi: hi wraps to 0 for the last tile of a 2^32 docID space)
                                        lc.visit(doc, f[t]);
                        }
                } else {
                        // tail block: (varbyte delta, varbyte freq) pairs (lucene_codec.cpp:527-550); lane-strided after a serial boundary walk
                        const uint32_t tail = T.documents & 127u;
                        const uint8_t *p;
                        if (len + 32u <= stageBytes) {
                                const uint32_t skew = stage_copy(ix.index, off, len, stage, lane);
                                __syncwarp();
                                p = stage + skew;
                        } else
                                p = ix.index + off;
                        if (lane == 0) {
                                uint32_t doc = prev;
                                for (uint32_t i = 0; i < tail; ++i) {
                                        doc += varbyte_get(p);
                                        const uint32_t fr = varbyte_get(p);
                                        if (doc >= lc.lo) {
                                                if (doc - lc.lo >= lc.hi - lc.lo)
                                                        break;
                                                lc.visit(doc, fr);
                                        }
                                }
                        }
                }
                __syncwarp();
        }
        if (lc.want_bits)
                lc.bits.flush();
}

// ------------------------------------------------------------------------------------------------ CTA utilities
// exclusive scan of one value per thread across the CTA; returns exclusive prefix, *total = sum
__device__ __forceinline__ uint32_t cta_excl_scan(uint32_t v, uint32_t *total, uint32_t *s_warp /*kWarps+1*/) {
        const int      lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        const uint32_t incl = warp_incl_scan(v, lane);
        __syncthreads();
        if (lane == 31)
                s_warp[warp] = incl;
        __syncthreads();
        uint32_t base = 0, tot = 0;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
                const uint32_t x = s_warp[w];
                if (w < warp)
                        base += x;
                tot += x;
        }
        *total = tot;
        return base + incl - v;
}

// descending bitonic sort of n2 (power of two) 64-bit keys in shared memory
__device__ void cta_bitonic_desc(unsigned long long *a, uint32_t n2) {
        for (uint32_t k2 = 2; k2 <= n2; k2 <<= 1) {
                for (uint32_t j = k2 >> 1; j > 0; j >>= 1) {
                        for (uint32_t i = threadIdx.x; i < n2; i += blockDim.x) {
                                const uint32_t p = i ^ j;
                                if (p > i) {
                                        const unsigned long long x = a[i], y = a[p];
                                        const bool               desc = (i & k2) == 0;
                                        if (desc ? (x < y) : (x > y)) {
                                                a[i] = y;
                                                a[p] = x;
                                        }
                                }
                        }
                        __syncthreads();
                }
        }
}

__device__ __forceinline__ uint32_t next_pow2(uint32_t v) {
        uint32_t p = 1;
        while (p < v)
                p <<= 1;
        return p;
}

// top-k key: (score bits << 32) | ~docid  — descending key order == (score desc, docID asc). scores are >= 0.
__device__ __forceinline__ unsigned long long make_key(float score, uint32_t doc) {
        return (static_cast<unsigned long long>(__float_as_uint(score)) << 32) | static_cast<unsigned long long>(~doc);
}

#include "phrase.cuh"

// ------------------------------------------------------------------------------------------------ the fused kernel
extern __shared__ __align__(16) uint8_t dyn_smem[];

// the documents of word wi (docIDs [32 wi, 32 wi + 32)) that a query's filter keeps: in its allow set (if it has one) and not in its deny
// set (IndexDocumentsFilter::filter, exec.cpp:1108-1116).  Only the filtered instantiations (FILT) call it.
__device__ __forceinline__ uint32_t filter_keep(const DevFilter &F, uint32_t wi) {
        uint32_t k = 0xffffffffu;
        if (F.allow)
                k = __ldg(F.allow + wi);
        if (F.deny)
                k &= ~__ldg(F.deny + wi);
        return k;
}

// PH: the instantiation that also executes OP_PHRASE (position checks, phrase.cuh) — used only for batches that hold phrase nodes, so that
// the cursor code costs the common instantiation neither registers nor a stack frame.  FILT: likewise for batches that hold a query with a
// document filter (ExecParams::filters)
template <bool PH, bool FILT> __global__ void __launch_bounds__(kThreads) k_exec_tiles(ExecParams P) {
        const uint32_t W     = 1u << P.exec_shift;
        const uint32_t NW    = W >> 5; // bitmap words per slot
        const bool     scored = P.mode != 0;
        // shared memory carve-up
        uint32_t *slots = reinterpret_cast<uint32_t *>(dyn_smem);                                   // nslots * NW words
        float *   acc   = reinterpret_cast<float *>(dyn_smem + size_t(P.nslots) * NW * 4);         // W floats (scored only)
        uint8_t * stage = dyn_smem + size_t(P.nslots) * NW * 4 + (scored ? size_t(W) * 4 : 0);     // kWarps * P.stage_bytes
        unsigned long long *list = reinterpret_cast<unsigned long long *>(stage + kWarps * P.stage_bytes); // kTileListCap keys (top-k only)

        __shared__ uint32_t s_item, s_warp[kWarps + 1], s_misc[4], s_n;
        __shared__ float    s_lut[64];
        __shared__ unsigned long long s_base;

        const int tid = threadIdx.x, lane = tid & 31;

        for (;;) {
                __syncthreads();
                if (tid == 0)
                        s_item = atomicAdd(P.ticket, 1u);
                __syncthreads();
                const uint32_t gitem = s_item; // ticket: the kernel's own item space (queries taken by k_score_flat own no tickets)
                if (gitem >= P.gen_items)
                        break;
                // locate the query: last q with gen_base <= gitem
                uint32_t qlo = 0, qhi = P.nq;
                while (qhi - qlo > 1) {
                        const uint32_t mid = (qlo + qhi) >> 1;
                        if (P.queries[mid].gen_base <= gitem)
                                qlo = mid;
                        else
                                qhi = mid;
                }
                const uint32_t q    = qlo;
                const DevQuery Q    = P.queries[q];
                const uint32_t item = Q.item_base + (gitem - Q.gen_base); // batch-wide (query, tile) item: index of the segment arrays
                const uint32_t tile = Q.tile_lo + (item - Q.item_base);
                const uint32_t lo = tile << P.exec_shift, hi = lo + W;

                if (scored) {
                        for (uint32_t i = tid; i < W; i += kThreads)
                                acc[i] = 0.f;
                }
                bool dead = false;

                for (uint32_t si = 0; si < Q.nsteps && !dead; ++si) {
                        const DevStep st  = P.steps[Q.step_begin + si];
                        uint32_t *    dst = slots + size_t(st.dst) * NW;
                        __syncthreads();
                        if (st.op == OP_CLEAR) {
                                for (uint32_t i = tid; i < NW; i += kThreads)
                                        dst[i] = 0;
                        } else if (st.op == OP_SLOT) {
                                const uint32_t *src = slots + size_t(st.src) * NW;
                                for (uint32_t i = tid; i < NW; i += kThreads) {
                                        const uint32_t s = src[i];
                                        if (st.mode == M_SET) dst[i] = s;
                                        else if (st.mode == M_OR) dst[i] |= s;
                                        else if (st.mode == M_AND) dst[i] &= s;
                                        else if (st.mode == M_ANDNOT) dst[i] &= ~s;
                                }
                        } else if (st.op == OP_COUNT_ADD) {
                                // bit-sliced saturating counters: plane j of the counter lives in slot dst + j
                                const uint32_t *src = slots + size_t(st.src) * NW;
                                for (uint32_t i = tid; i < NW; i += kThreads) {
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
                                for (uint32_t i = tid; i < NW; i += kThreads) {
                                        uint32_t gt = 0, eq = 0xffffffffu;
                                        for (int j = int(st.mode) - 1; j >= 0; --j) {
                                                const uint32_t p = slots[size_t(st.src + j) * NW + i];
                                                if ((m >> j) & 1u) eq &= p;
                                                else gt |= eq & p;
                                        }
                                        dst[i] = gt | eq;
                                }
                        } else if (st.op == OP_PHRASE) {
                                // position filter over the candidates of dst (+ the phrase's score where it holds); phrase.cuh
                                if constexpr (PH)
                                        phrase_check(P.ix, P.steps + Q.step_begin + si + 1u, st.mode, lo, NW, dst, (scored && (st.flags & F_SCORE)) ? acc : nullptr, st.idf, tid, kThreads);
                        } else if (st.op == OP_ARG) {
                                // operand words of the preceding step
                        } else {
                                // OP_LEAF / OP_LEAFSCORE
                                const bool     second   = st.op == OP_LEAFSCORE;
                                const int      mode     = second ? M_NONE : st.mode;
                                const bool     doScore  = second || (st.flags & F_SCORE);
                                uint32_t *     tmp      = slots + size_t(P.nslots - 1) * NW; // scratch slot (AND)
                                const bool     haveTerm = st.term != kEmptyTerm;
                                DevTerm        T;
                                uint32_t       bA = 1, bB = 0;
                                if (haveTerm) {
                                        T = P.ix.terms[st.term];
                                        tile_block_range(P.ix, T, lo, W, bA, bB);
                                }
                                // prepare destination
                                if (mode == M_SET) {
                                        for (uint32_t i = tid; i < NW; i += kThreads)
                                                dst[i] = 0;
                                } else if (mode == M_AND) {
                                        for (uint32_t i = tid; i < NW; i += kThreads)
                                                tmp[i] = 0;
                                        // narrow the block range to the span of candidates still alive in dst (skip == advance())
                                        uint32_t mn = 0xffffffffu, mx = 0;
                                        for (uint32_t i = tid; i < NW; i += kThreads) {
                                                const uint32_t w = dst[i];
                                                if (w) {
                                                        mn = min(mn, i * 32u + uint32_t(__ffs(int(w)) - 1));
                                                        mx = max(mx, i * 32u + uint32_t(31 - __clz(int(w))));
                                                }
                                        }
                                        for (int d = 16; d > 0; d >>= 1) {
                                                mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, d));
                                                mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
                                        }
                                        if (tid == 0) {
                                                s_misc[0] = 0xffffffffu;
                                                s_misc[1] = 0;
                                        }
                                        __syncthreads();
                                        if (lane == 0) {
                                                atomicMin(&s_misc[0], mn);
                                                atomicMax(&s_misc[1], mx);
                                        }
                                        __syncthreads();
                                        mn = s_misc[0];
                                        mx = s_misc[1];
                                        if (mn == 0xffffffffu) {
                                                bA = 1;
                                                bB = 0; // dst is empty: nothing can survive
                                        } else if (bA <= bB) {
                                                if (tid == 0) {
                                                        const uint32_t *bl = P.ix.blk_last + T.dir_begin;
                                                        const uint32_t  dmin = lo + mn, dmax = lo + mx;
                                                        uint32_t        a = bA, b = bB;
                                                        // first block with last >= dmin
                                                        uint32_t l = a, r = b + 1;
                                                        while (l < r) {
                                                                const uint32_t m = (l + r) >> 1;
                                                                if (bl[m] < dmin) l = m + 1;
                                                                else r = m;
                                                        }
                                                        a = l;
                                                        // first block with last >= dmax
                                                        l = a;
                                                        r = b + 1;
                                                        while (l < r) {
                                                                const uint32_t m = (l + r) >> 1;
                                                                if (bl[m] < dmax) l = m + 1;
                                                                else r = m;
                                                        }
                                                        b         = min(l, b);
                                                        s_misc[2] = a;
                                                        s_misc[3] = b;
                                                }
                                                __syncthreads();
                                                bA = s_misc[2];
                                                bB = s_misc[3];
                                        }
                                }
                                if (doScore && tid < 64)
                                        s_lut[tid] = bm25_score(st.idf, uint32_t(tid));
                                __syncthreads();

                                if (haveTerm && bA <= bB) {
                                        LeafCtx lc;
                                        lc.lo         = lo;
                                        lc.hi         = hi;
                                        lc.want_bits  = mode != M_NONE;
                                        lc.want_score = doScore;
                                        lc.acc        = acc;
                                        lc.lut        = s_lut;
                                        lc.mask       = second ? (slots + size_t(st.src) * NW) : nullptr;
                                        lc.idf        = st.idf;
                                        const uint32_t *skipfilt = nullptr;
                                        if (mode == M_AND) {
                                                lc.bits.init(tmp, dst, M_OR);
                                                skipfilt = dst;
                                        } else if (mode == M_ANDNOT) {
                                                lc.bits.init(dst, nullptr, M_ANDNOT);
                                                skipfilt = dst; // nothing to clear where dst is already empty
                                        } else
                                                lc.bits.init(dst, nullptr, M_OR);
                                        if (P.ix.codec == 0) {
                                                if (doScore) google_leaf<true>(P.ix, T, bA, bB, lc, skipfilt, stage, P.stage_bytes);
                                                else google_leaf<false>(P.ix, T, bA, bB, lc, skipfilt, stage, P.stage_bytes);
                                        } else {
                                                if (doScore) lucene_leaf<true>(P.ix, T, bA, bB, lc, skipfilt, stage, P.stage_bytes);
                                                else lucene_leaf<false>(P.ix, T, bA, bB, lc, skipfilt, stage, P.stage_bytes);
                                        }
                                }
                                if (mode == M_AND) {
                                        __syncthreads();
                                        for (uint32_t i = tid; i < NW; i += kThreads)
                                                dst[i] = tmp[i];
                                }
                        }
                        if (st.flags & F_BREAK_IF_EMPTY) {
                                __syncthreads();
                                uint32_t any = 0;
                                for (uint32_t i = tid; i < NW; i += kThreads)
                                        any |= dst[i];
                                if (__syncthreads_or(int(any != 0)) == 0)
                                        dead = true;
                        }
                }
                __syncthreads();

                // masked documents (masked_documents_registry::test, exec.cpp:1108-1116) never reach the sink / the top-k
                if (!dead && P.ix.masked) {
                        uint32_t *      r  = slots + size_t(Q.root_slot) * NW;
                        const uint32_t *mk = P.ix.masked + (lo >> 5);
                        for (uint32_t i = tid; i < NW; i += kThreads)
                                r[i] &= ~mk[i];
                        __syncthreads();
                }
                // ... and neither do the documents the query's filter drops: they take no top-k candidate slot and never move theta
                if constexpr (FILT) {
                        if (!dead) {
                                const DevFilter F = P.filters[q];
                                uint32_t *      r = slots + size_t(Q.root_slot) * NW;
                                for (uint32_t i = tid; i < NW; i += kThreads)
                                        r[i] &= filter_keep(F, (lo >> 5) + i);
                                __syncthreads();
                        }
                }
                // ---------------------------------------------------------------- emission
                const uint32_t *root = slots + size_t(Q.root_slot) * NW;
                if (dead) {
                        if (P.mode != 2 && tid == 0) {
                                P.item_off[item] = 0;
                                P.item_cnt[item] = 0;
                        }
                        continue;
                }
                if (P.mode != 2) {
                        // DOCS_ONLY / SCORED_ALL: ordered compaction of the root docset; thread t owns words [t*wpt, (t+1)*wpt)
                        const uint32_t wpt = NW / kThreads;
                        uint32_t       c   = 0;
                        for (uint32_t i = 0; i < wpt; ++i)
                                c += __popc(root[tid * wpt + i]);
                        uint32_t       total;
                        const uint32_t excl = cta_excl_scan(c, &total, s_warp);
                        if (tid == 0) {
                                unsigned long long base = 0;
                                if (total) {
                                        base = atomicAdd(P.seg_cursor, static_cast<unsigned long long>(total));
                                        atomicAdd(&P.match_counts[q], static_cast<unsigned long long>(total));
                                        if (base + total > P.seg_capacity) {
                                                *P.overflow = 1;
                                                base        = ~0ull;
                                        }
                                }
                                s_base           = base;
                                P.item_off[item] = base;
                                P.item_cnt[item] = base == ~0ull ? 0 : total;
                        }
                        __syncthreads();
                        const unsigned long long base = s_base;
                        if (total && base != ~0ull) {
                                unsigned long long pos = base + excl;
                                for (uint32_t i = 0; i < wpt; ++i) {
                                        const uint32_t wi = tid * wpt + i;
                                        uint32_t       w  = root[wi];
                                        while (w) {
                                                const uint32_t bit = uint32_t(__ffs(int(w)) - 1);
                                                w &= w - 1;
                                                const uint32_t rel = wi * 32u + bit;
                                                P.seg_docids[pos]  = lo + rel;
                                                if (scored)
                                                        P.seg_scores[pos] = acc[rel];
                                                ++pos;
                                        }
                                }
                        }
                } else {
                        // SCORED_TOPK: keep the tile's candidates whose score can still reach the query's top-k
                        const uint32_t k = P.k;
                        if (tid == 0)
                                s_n = 0;
                        unsigned long long thr = static_cast<unsigned long long>(*reinterpret_cast<volatile uint32_t *>(&P.theta[q])) << 32;
                        uint32_t           matches = 0;
                        const uint32_t     rounds  = W / 512u;
                        for (uint32_t r = 0; r < rounds; ++r) {
                                __syncthreads();
                                // 512 docs per round: thread t looks at nibble (t&7) of word r*16 + (t>>3); list holds <= k + 512 <= kTileListCap keys
                                const uint32_t wi   = r * 16u + (uint32_t(tid) >> 3);
                                uint32_t       bits = (root[wi] >> ((tid & 7) * 4)) & 0xfu;
                                matches += __popc(bits);
                                while (bits) {
                                        const uint32_t bit = uint32_t(__ffs(int(bits)) - 1);
                                        bits &= bits - 1;
                                        const uint32_t rel = wi * 32u + (tid & 7) * 4u + bit;
                                        const unsigned long long key = make_key(acc[rel], lo + rel);
                                        if (key >= thr) {
                                                const uint32_t idx = atomicAdd(&s_n, 1u);
                                                list[idx]          = key;
                                        }
                                }
                                __syncthreads();
                                const uint32_t n = s_n;
                                if (n > k) {
                                        const uint32_t n2 = next_pow2(n);
                                        for (uint32_t i = n + tid; i < n2; i += kThreads)
                                                list[i] = 0ull;
                                        __syncthreads();
                                        cta_bitonic_desc(list, n2);
                                        thr = max(thr, list[k - 1]);
                                        __syncthreads();
                                        if (tid == 0)
                                                s_n = k;
                                }
                        }
                        __syncthreads();
                        // per-query match count
                        for (int d = 16; d > 0; d >>= 1)
                                matches += __shfl_xor_sync(0xffffffffu, matches, d);
                        if (lane == 0 && matches)
                                atomicAdd(&P.match_counts[q], static_cast<unsigned long long>(matches));
                        const uint32_t n = s_n;
                        if (n) {
                                if (tid == 0)
                                        s_misc[0] = atomicAdd(&P.cand_cursor[q], n);
                                __syncthreads();
                                const uint32_t cb = s_misc[0];
                                for (uint32_t i = tid; i < n; i += kThreads) {
                                        const unsigned long long key = list[i];
                                        if (cb + i < Q.cand_cap)
                                                P.cand[size_t(Q.cand_base) + cb + i] = make_uint2(uint32_t(key >> 32), ~uint32_t(key));
                                }
                                if (n >= k && tid == 0) {
                                        // after a prune list[] is sorted; n == k exactly then. The k-th best of this tile bounds the query's k-th best from below.
                                        atomicMax(&P.theta[q], uint32_t(thr >> 32));
                                }
                        }
                }
        }
}

#include "score_flat.cuh"
#include "exec_docs.cuh"

// ------------------------------------------------------------------------------------------------ segment ordering
// one CTA per query: exclusive scan of the per-tile match counts -> destination offset of every tile segment
__global__ void __launch_bounds__(kThreads) k_item_scan(const DevQuery *queries, const uint32_t *item_cnt, const uint64_t *q_offsets, uint64_t *item_dst) {
        __shared__ uint32_t s_warp[kWarps + 1];
        const DevQuery      Q    = queries[blockIdx.x];
        uint64_t            run  = q_offsets[blockIdx.x];
        for (uint32_t base = 0; base < Q.ntiles; base += kThreads) {
                const uint32_t i = base + threadIdx.x;
                const uint32_t c = i < Q.ntiles ? item_cnt[Q.item_base + i] : 0u;
                uint32_t       total;
                const uint32_t ex = cta_excl_scan(c, &total, s_warp);
                if (i < Q.ntiles)
                        item_dst[Q.item_base + i] = run + ex;
                run += total;
                __syncthreads();
        }
}

// single CTA: exclusive scan of per-query match counts
__global__ void __launch_bounds__(kThreads) k_query_scan(const unsigned long long *match_counts, uint32_t nq, uint64_t *q_offsets) {
        __shared__ unsigned long long s_part[kThreads];
        // sequential chunks per thread (nq is small: a few thousand)
        const uint32_t per = (nq + kThreads - 1) / kThreads;
        const uint32_t b = threadIdx.x * per, e = min(nq, b + per);
        unsigned long long s = 0;
        for (uint32_t i = b; i < e; ++i)
                s += match_counts[i];
        s_part[threadIdx.x] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
                unsigned long long run = 0;
                for (int i = 0; i < kThreads; ++i) {
                        const unsigned long long v = s_part[i];
                        s_part[i]                  = run;
                        run += v;
                }
                q_offsets[nq] = run;
        }
        __syncthreads();
        unsigned long long run = s_part[threadIdx.x];
        for (uint32_t i = b; i < e; ++i) {
                q_offsets[i] = run;
                run += match_counts[i];
        }
}

// one warp per work item: copy its segment to its final (query-ordered) position
__global__ void __launch_bounds__(kThreads) k_gather(uint32_t total_items, const uint64_t *item_off, const uint32_t *item_cnt, const uint64_t *item_dst,
                                                     const uint32_t *seg_docids, const float *seg_scores, uint32_t *out_docids, float *out_scores) {
        const uint32_t item = blockIdx.x * kWarps + (threadIdx.x >> 5);
        if (item >= total_items)
                return;
        const uint32_t n = item_cnt[item];
        if (!n)
                return;
        const uint64_t s = item_off[item], d = item_dst[item];
        for (uint32_t i = threadIdx.x & 31; i < n; i += 32) {
                out_docids[d + i] = seg_docids[s + i];
                if (seg_scores)
                        out_scores[d + i] = seg_scores[s + i];
        }
}

// ------------------------------------------------------------------------------------------------ top-k select / merge
// one CTA per query over its candidates (score bits, docid); exact (score desc, docID asc) top-k
__global__ void __launch_bounds__(kThreads) k_topk_select(const DevQuery *queries, const uint2 *cand, const uint32_t *cand_cursor, uint32_t k,
                                                          uint32_t *out_docids, float *out_scores, uint32_t *out_counts) {
        __shared__ unsigned long long list[kListCap];
        const uint32_t                q    = blockIdx.x;
        const DevQuery                Q    = queries[q];
        const uint32_t                n    = min(cand_cursor[q], Q.cand_cap);
        const uint2 *                 c    = cand + size_t(Q.cand_base);
        uint32_t                      kept = 0;
        const uint32_t                chunk = kListCap - k;
        for (uint32_t base = 0; base < n; base += chunk) {
                const uint32_t m = min(chunk, n - base);
                for (uint32_t i = threadIdx.x; i < m; i += kThreads) {
                        const uint2 e  = c[base + i];
                        list[kept + i] = (static_cast<unsigned long long>(e.x) << 32) | static_cast<unsigned long long>(~e.y);
                }
                const uint32_t tot = kept + m, n2 = next_pow2(tot);
                for (uint32_t i = tot + threadIdx.x; i < n2; i += kThreads)
                        list[i] = 0ull;
                __syncthreads();
                cta_bitonic_desc(list, n2);
                kept = min(tot, k);
                __syncthreads();
        }
        for (uint32_t i = threadIdx.x; i < k; i += kThreads) {
                if (i < kept) {
                        const unsigned long long key  = list[i];
                        out_docids[size_t(q) * k + i] = ~uint32_t(key);
                        out_scores[size_t(q) * k + i] = __uint_as_float(uint32_t(key >> 32));
                } else {
                        out_docids[size_t(q) * k + i] = 0;
                        out_scores[size_t(q) * k + i] = -1.0f; // padding (real scores are >= 0)
                }
        }
        if (threadIdx.x == 0)
                out_counts[q] = kept;
}

// one CTA per query: merge nshards top-k lists laid out [shard][nq][k]
__global__ void __launch_bounds__(kThreads) k_topk_merge(const uint32_t *docids, const float *scores, uint32_t nshards, uint32_t nq, uint32_t k,
                                                         uint32_t *out_docids, float *out_scores) {
        __shared__ unsigned long long list[kListCap];
        const uint32_t                q    = blockIdx.x;
        uint32_t                      kept = 0;
        const uint32_t                per  = max(1u, (kListCap - k) / k); // shards per round
        for (uint32_t s0 = 0; s0 < nshards; s0 += per) {
                const uint32_t ns = min(per, nshards - s0), m = ns * k;
                for (uint32_t i = threadIdx.x; i < m; i += kThreads) {
                        const uint32_t s = s0 + i / k, j = i % k;
                        const size_t   at = (size_t(s) * nq + q) * k + j;
                        const float    sc = scores[at];
                        list[kept + i]    = sc < 0.f ? 0ull : make_key(sc, docids[at]);
                }
                const uint32_t tot = kept + m, n2 = next_pow2(tot);
                for (uint32_t i = tot + threadIdx.x; i < n2; i += kThreads)
                        list[i] = 0ull;
                __syncthreads();
                cta_bitonic_desc(list, n2);
                kept = min(tot, k);
                __syncthreads();
        }
        for (uint32_t i = threadIdx.x; i < k; i += kThreads) {
                const unsigned long long key = i < kept ? list[i] : 0ull;
                if (key) {
                        out_docids[size_t(q) * k + i] = ~uint32_t(key);
                        out_scores[size_t(q) * k + i] = __uint_as_float(uint32_t(key >> 32));
                } else {
                        out_docids[size_t(q) * k + i] = 0;
                        out_scores[size_t(q) * k + i] = -1.0f;
                }
        }
}

#include "decode_stream.cuh"
#include "encode_google.cuh"
#include "encode_lucene.cuh"
#include "collect.cuh"
#include "intersect.cuh"
#include "percolate.cuh"
#include "percolate_update.cuh"
#include "index_docs.cuh"
#include "merge.cuh"

// ------------------------------------------------------------------------------------------------ launch wrappers
uint32_t exec_stage_bytes(int codec) {
        // per-warp staging of k_exec_tiles: Google copies the byte span of 32 blocks; one Lucene block is at most 2*(1+4*255) bytes
        return codec == 0 ? kStageBytes : 3072u; // 2560 block bytes + 512 exception scratch
}

size_t exec_smem_bytes(uint32_t tile_shift, uint32_t nslots, int mode, int codec) {
        const size_t W = size_t(1) << tile_shift;
        size_t       s = size_t(nslots) * (W / 32) * 4 + size_t(kWarps) * exec_stage_bytes(codec);
        if (mode != 0)
                s += W * 4;
        if (mode == 2)
                s += size_t(kTileListCap) * 8;
        return s;
}

cudaError_t launch_exec_tiles(const ExecParams &P, int grid, cudaStream_t stream) {
        const size_t smem = exec_smem_bytes(P.exec_shift, P.nslots, P.mode, P.ix.codec);
        const void * fn   = P.filters ? (P.has_phrase ? (const void *)k_exec_tiles<true, true> : (const void *)k_exec_tiles<false, true>)
                                      : (P.has_phrase ? (const void *)k_exec_tiles<true, false> : (const void *)k_exec_tiles<false, false>);
        cudaError_t  e    = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
        if (e != cudaSuccess)
                return e;
        void *args[] = {(void *)&P};
        return cudaLaunchKernel(fn, dim3(grid), dim3(kThreads), args, smem, stream);
}

int exec_max_ctas_per_sm(uint32_t tile_shift, uint32_t nslots, int mode, int codec, bool filt) {
        const size_t smem = exec_smem_bytes(tile_shift, nslots, mode, codec);
        // (the phrase instantiation needs at least as many registers: size the grid for it when in doubt — a smaller grid is still correct)
        const void *a = filt ? (const void *)k_exec_tiles<false, true> : (const void *)k_exec_tiles<false, false>;
        const void *b = filt ? (const void *)k_exec_tiles<true, true> : (const void *)k_exec_tiles<true, false>;
        if (cudaFuncSetAttribute(a, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess ||
            cudaFuncSetAttribute(b, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess)
                return 0;
        int n = 0, m = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, a, kThreads, smem) != cudaSuccess ||
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&m, b, kThreads, smem) != cudaSuccess)
                return 0;
        return std::min(n, m);
}

cudaError_t launch_query_scan(const unsigned long long *match_counts, uint32_t nq, uint64_t *q_offsets, cudaStream_t stream) {
        k_query_scan<<<1, kThreads, 0, stream>>>(match_counts, nq, q_offsets);
        return cudaGetLastError();
}

cudaError_t launch_item_scan(const DevQuery *queries, uint32_t nq, const uint32_t *item_cnt, const uint64_t *q_offsets, uint64_t *item_dst, cudaStream_t stream) {
        k_item_scan<<<nq, kThreads, 0, stream>>>(queries, item_cnt, q_offsets, item_dst);
        return cudaGetLastError();
}

cudaError_t launch_gather(uint32_t total_items, const uint64_t *item_off, const uint32_t *item_cnt, const uint64_t *item_dst, const uint32_t *seg_docids,
                          const float *seg_scores, uint32_t *out_docids, float *out_scores, cudaStream_t stream) {
        if (!total_items)
                return cudaSuccess;
        const uint32_t grid = (total_items + kWarps - 1) / kWarps;
        k_gather<<<grid, kThreads, 0, stream>>>(total_items, item_off, item_cnt, item_dst, seg_docids, seg_scores, out_docids, out_scores);
        return cudaGetLastError();
}

cudaError_t launch_topk_select(const DevQuery *queries, uint32_t nq, const uint2 *cand, const uint32_t *cand_cursor, uint32_t k, uint32_t *out_docids,
                               float *out_scores, uint32_t *out_counts, cudaStream_t stream) {
        k_topk_select<<<nq, kThreads, 0, stream>>>(queries, cand, cand_cursor, k, out_docids, out_scores, out_counts);
        return cudaGetLastError();
}

cudaError_t launch_topk_merge(const uint32_t *docids, const float *scores, uint32_t nshards, uint32_t nq, uint32_t k, uint32_t *out_docids, float *out_scores,
                              cudaStream_t stream) {
        k_topk_merge<<<nq, kThreads, 0, stream>>>(docids, scores, nshards, nq, k, out_docids, out_scores);
        return cudaGetLastError();
}

// Load time: the bitmaps of the dense and the probe tier (DevIndex::dense at probe_off, zeroed by the caller).  One thread per block of a selected term: it walks the
// block's doc-delta section (the deltas of documents 2..n, the block's last docID comes from the directory) and ORs one word per 32
// docIDs it touched.  blk_prefix[s] = blocks of the selected terms before sel[s] (nsel + 1 entries).
__global__ void __launch_bounds__(kThreads) k_build_dense(DevIndex ix, const uint32_t *sel, const unsigned long long *blk_prefix, uint32_t nsel,
                                                           unsigned long long total_blocks, uint32_t *dense) {
        const unsigned long long g = blockIdx.x * 1ull * blockDim.x + threadIdx.x;
        if (g >= total_blocks)
                return;
        uint32_t lo = 0, hi = nsel; // the selected term whose blocks hold g: blk_prefix[lo] <= g < blk_prefix[lo + 1]
        while (hi - lo > 1u) {
                const uint32_t mid = (lo + hi) >> 1;
                if (blk_prefix[mid] <= g) lo = mid;
                else hi = mid;
        }
        const uint32_t  t = sel[lo], b = uint32_t(g - blk_prefix[lo]);
        const DevTerm   T = ix.terms[t];
        const uint32_t *bl = ix.blk_last + T.dir_begin;
        const uint32_t  base = (T.first_doc >> kDenseAlignShift) << kDenseAlignShift;
        uint32_t *      bm   = dense + ix.probe_off[t];
        const uint32_t  n    = (b + 1u == T.nblocks) ? (T.documents - 32u * (T.nblocks - 1u)) : 32u;
        const uint8_t * p    = ix.index + ix.blk_off[T.dir_begin + b];
        uint32_t        doc = b ? bl[b - 1] : 0u, cw = 0xffffffffu, cur = 0;
        for (uint32_t i = 0; i < n; ++i) {
                doc               = i + 1u < n ? doc + varbyte_get(p) : bl[b];
                const uint32_t w  = (doc - base) >> 5;
                if (w != cw && cur)
                        atomicOr(bm + cw, cur);
                cur = (w != cw ? 0u : cur) | (1u << (doc & 31u));
                cw  = w;
        }
        if (cur)
                atomicOr(bm + cw, cur);
}

cudaError_t launch_build_dense(const DevIndex &ix, const uint32_t *sel, const unsigned long long *blk_prefix, uint32_t nsel, uint64_t total_blocks,
                               uint32_t *dense, cudaStream_t stream) {
        if (!total_blocks)
                return cudaSuccess;
        const unsigned grid = unsigned((total_blocks + kThreads - 1) / kThreads);
        k_build_dense<<<grid, kThreads, 0, stream>>>(ix, sel, blk_prefix, nsel, total_blocks, dense);
        return cudaGetLastError();
}

uint32_t kernel_max_k() {
        return kMaxK;
}

} // namespace trn
