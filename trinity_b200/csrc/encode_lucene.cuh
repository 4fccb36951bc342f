// GPU-side Encoder for the LUCENE postings layout (SURVEY.md 8(f) row 4, the second codec).  (Included by kernels.cu after
// encode_google.cuh, whose varbyte helpers and scan it uses.)
//
// Replaces (reference): Codecs::Lucene::Encoder begin_term / begin_document / new_hit / end_document / end_term
// (lucene_codec.cpp:163-388; the int-block is FastPFor<4>::encodeArray of one 128-value page, fastpfor.h:143-271).  The bytes are the
// ones this repo's host encoder writes (codecs.cpp), pinned by tests/test_gpu_encoder_lucene.py (no payloads) and tests/test_gpu_payloads.py
// (payloads); where the reference leaves the PFor byte container's padding uninitialised, both write zeros.
//
//   int-block = 00 varbyte(v)                                   all 128 values equal
//             | u8 L, L words: 128 | wheremeta | 4 x 32 values at b bits | nb | {b, cexcept, [maxb, exception positions]} padded
//                              | exception bitmap | [count | the exceptions' high bits at k = maxb - b bits]   (k >= 2 only)
//   chunk     = u32 hitsDataOffset, u32 sumHits, u32 positionsChunkSize, u16 skiplistSize
//             | full blocks: intblock(docID deltas) intblock(freqs) | tail: varbyte(delta) varbyte(freq) per document
//             | one 22-byte skiplist entry per full block (at most 65535)
//   hits.data = per term, its hits in posting order cut into blocks of 128 that cross documents:
//               full block: intblock(position deltas) 00 00 00 (payload sizes all 0, no payload bytes) | tail: varbyte(delta << 1) per hit
//               with payloads (the PAYLOADS instantiation of k_enc_lucene_hits): full block: intblock(position deltas) intblock(payload
//               sizes) varbyte(sum of the sizes) the payload bytes | tail: varbyte(delta << 1 | changed) [u8 size when changed] per hit, then
//               every payload byte of the tail; `changed` compares with the previous hit of the tail, across documents (0 before the first)
// A block's bytes depend on nothing but its own values, so (1) one warp per unit (a full block, or a term's tail) computes its size,
// (2) exclusive scans place the units, (3) one warp per unit writes it; the warp of a term's doc tail writes the chunk header, lane 0 of
// a full doc block's warp its skiplist entry.  Lane l holds values l, 32 + l, 64 + l, 96 + l of a unit.
#pragma once

static constexpr uint32_t kLucBlock     = 128; // Codecs::Lucene::BLOCK_SIZE
static constexpr uint32_t kLucPageWords = 168; // largest PFor page: 3 + 33 (byte container) + 2 + 4 maxb (values + exceptions) = 166
static constexpr uint32_t kLucSkipEntry = 22;  // u32 x 5 + u16

struct LucIntBlock {
        uint32_t bytes;              // of the whole int-block, length byte included
        uint32_t b, maxb, cexcept, L; // L: page words (0: all values equal)
        uint32_t v0;
};

// FastPFor<4>::getBestBFromData (fastpfor.h:143-171) + the size of the int-block.  The host scans bb = maxb-1 .. 0 and keeps a candidate
// only when it is strictly cheaper: the minimum cost, ties to the larger b, the initial b = maxb winning every tie.  Lane bb evaluates
// candidate bb; one min-reduction over (cost, 63 - b) picks the same b.  hist: 33 words of the warp's shared memory.
__device__ __forceinline__ LucIntBlock luc_plan(const uint32_t (&v)[4], int lane, uint32_t *hist) {
        LucIntBlock P{};
        P.v0     = __shfl_sync(0xffffffffu, v[0], 0);
        const bool eq = __all_sync(0xffffffffu, v[0] == P.v0 && v[1] == P.v0 && v[2] == P.v0 && v[3] == P.v0);
        if (eq) {
                P.bytes = 1u + vb_len_of(P.v0);
                return P;
        }
        hist[lane] = 0;
        if (lane == 0)
                hist[32] = 0;
        __syncwarp();
        uint32_t mb = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
                const uint32_t bits = 32u - uint32_t(__clz(v[q]));
                atomicAdd(&hist[bits], 1u);
                mb = max(mb, bits);
        }
        const uint32_t maxb = __reduce_max_sync(0xffffffffu, mb);
        __syncwarp();
        uint32_t c = hist[lane + 1]; // -> cexcept(lane): values with more than `lane` bits
        for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_down_sync(0xffffffffu, c, o);
                if (lane + o < 32)
                        c += y;
        }
        __syncwarp(); // hist is reused by the next int-block of the warp
        uint32_t key = 0xffffffffu;
        if (uint32_t(lane) < maxb) {
                const uint32_t bb   = uint32_t(lane);
                uint32_t       cost = c * 8u + c * (maxb - bb) + bb * kLucBlock + 8u;
                if (maxb - bb == 1u)
                        cost -= c;
                key = (cost << 6) | (63u - bb);
        }
        key                = min(__reduce_min_sync(0xffffffffu, key), ((maxb * kLucBlock) << 6) | (63u - maxb));
        P.b                = 63u - (key & 63u);
        P.maxb             = maxb;
        const uint32_t ce  = __shfl_sync(0xffffffffu, c, int(P.b & 31u));
        P.cexcept          = P.b == maxb ? 0u : ce;
        const uint32_t nb  = 2u + (P.cexcept ? 1u + P.cexcept : 0u);
        const uint32_t k   = maxb - P.b;
        uint32_t       L   = 2u + 4u * P.b + 1u + (nb + 3u) / 4u + 1u;
        if (P.cexcept && k >= 2u) {
                const uint32_t j = (P.cexcept + 31u) / 32u * 32u;
                L += 1u + j / 32u * k - (j - P.cexcept) * k / 32u;
        }
        P.L     = L;
        P.bytes = 1u + 4u * L;
        return P;
}

// OR `width` bits of v (already < 2^width) into the LSB-first bit stream w at bit `bit` (== pack32, codecs.cpp)
__device__ __forceinline__ void luc_or_bits(uint32_t *w, uint32_t bit, uint32_t v, uint32_t width) {
        const uint32_t i = bit >> 5, sh = bit & 31u;
        atomicOr(&w[i], v << sh);
        if (sh + width > 32u)
                atomicOr(&w[i + 1], v >> (32u - sh));
}

// writes the int-block planned by luc_plan at o (global memory); pg: kLucPageWords words of the warp's shared memory
__device__ void luc_write(uint8_t *o, const uint32_t (&v)[4], const LucIntBlock &P, int lane, uint32_t *pg) {
        if (!P.L) {
                if (lane == 0) {
                        o[0] = 0;
                        vb_store(o + 1, P.v0);
                }
                return;
        }
        const uint32_t b = P.b, k = P.maxb - P.b;
        for (uint32_t i = uint32_t(lane); i < P.L; i += 32u)
                pg[i] = 0;
        __syncwarp();
        const uint32_t meta = 2u + 4u * b; // the nb word
        const uint32_t nb   = 2u + (P.cexcept ? 1u + P.cexcept : 0u);
        const uint32_t bw   = meta + 1u + (nb + 3u) / 4u; // the exception bitmap word
        uint8_t *      by   = reinterpret_cast<uint8_t *>(pg + meta + 1u);
        const bool     bitmap = P.cexcept && k >= 2u;
        if (lane == 0) {
                pg[0]    = kLucBlock;
                pg[1]    = 1u + 4u * b; // wheremeta
                pg[meta] = nb;
                by[0]    = uint8_t(b);
                by[1]    = uint8_t(P.cexcept);
                if (P.cexcept)
                        by[2] = uint8_t(P.maxb);
                pg[bw] = bitmap ? 1u << (k - 1u) : 0u;
                if (bitmap)
                        pg[bw + 1] = P.cexcept;
        }
        const uint32_t m   = b == 32u ? 0xffffffffu : (1u << b) - 1u;
        uint32_t       run = 0; // exceptions in earlier lane groups
#pragma unroll
        for (int q = 0; q < 4; ++q) {
                const uint32_t i = uint32_t(q) * 32u + uint32_t(lane);
                if (b)
                        luc_or_bits(pg + 2, i * b, v[q] & m, b);
                const bool     exc  = b < 32u && (v[q] >> b) != 0u;
                const uint32_t ball = __ballot_sync(0xffffffffu, exc);
                if (exc) {
                        const uint32_t e = run + uint32_t(__popc(ball & ((1u << lane) - 1u)));
                        by[3 + e]        = uint8_t(i);
                        if (bitmap)
                                luc_or_bits(pg + bw + 2u, e * k, v[q] >> b, k);
                }
                run += uint32_t(__popc(ball));
        }
        __syncwarp();
        if (lane == 0)
                o[0] = uint8_t(P.L);
        const uint8_t *src = reinterpret_cast<const uint8_t *>(pg);
        for (uint32_t i = uint32_t(lane); i < 4u * P.L; i += 32u)
                o[1 + i] = src[i];
        __syncwarp(); // pg is reused by the next int-block of the warp
}

__device__ __forceinline__ void luc_put32(uint8_t *s, uint32_t v) {
        s[0] = uint8_t(v), s[1] = uint8_t(v >> 8), s[2] = uint8_t(v >> 16), s[3] = uint8_t(v >> 24);
}

// the unit's term: last term whose first unit is <= g (every term has at least one unit)
__device__ __forceinline__ uint32_t luc_term_of(const unsigned long long *unit_begin, uint32_t nterms, uint64_t g) {
        uint32_t lo = 0, hi = nterms - 1u;
        while (lo < hi) {
                const uint32_t mid = (lo + hi + 1u) >> 1;
                if (unit_begin[mid] <= g)
                        lo = mid;
                else
                        hi = mid - 1u;
        }
        return lo;
}

// size (WRITE = false) or bytes (WRITE = true) of one doc unit, one warp per unit
template <bool WRITE> __global__ void __launch_bounds__(128) k_enc_lucene_docs(EncLuceneParams E) {
        __shared__ uint32_t s_pg[4][kLucPageWords];
        __shared__ uint32_t s_hist[4][33];
        const int           warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const uint64_t      g    = uint64_t(blockIdx.x) * 4u + uint64_t(warp);
        if (g >= E.ndunits)
                return;
        uint32_t t;
        if (!WRITE) {
                t = luc_term_of(E.dunit_begin, E.nterms, g);
                if (lane == 0)
                        E.dterm[g] = t;
        } else
                t = E.dterm[g];
        const uint64_t tb = E.term_begin[t], te = E.term_begin[t + 1];
        const uint64_t u0 = E.dunit_begin[t], j = g - u0, nfull = (te - tb) / kLucBlock;
        const uint64_t d0 = tb + j * kLucBlock;
        const uint32_t n  = j < nfull ? kLucBlock : uint32_t((te - tb) % kLucBlock);
        uint32_t       dl[4], fr[4];
        bool           bad = false;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
                const uint32_t i = uint32_t(q) * 32u + uint32_t(lane);
                dl[q] = fr[q] = 0;
                if (i < n) {
                        const uint32_t d = E.docids[d0 + i], p = d0 + i == tb ? 0u : E.docids[d0 + i - 1];
                        bad |= d <= p; // also docID 0: lucene_codec.cpp begin_document
                        dl[q] = d - p;
                        fr[q] = E.freqs[d0 + i];
                }
        }
        if (__any_sync(0xffffffffu, bad)) {
                if (lane == 0) {
                        atomicExch(E.error, 1u);
                        if (!WRITE)
                                E.dsz[g] = 0;
                }
                return;
        }
        const uint64_t chunk = WRITE ? E.term_off[t] : 0u;
        const uint64_t base  = WRITE ? E.doff[u0] : 0u;
        uint8_t *      o     = WRITE ? E.index_out + chunk + 14u + (E.doff[g] - base) : nullptr;
        if (j < nfull) { // a full block: intblock(deltas) intblock(freqs) + its skiplist entry
                const LucIntBlock pd = luc_plan(dl, lane, s_hist[warp]);
                const LucIntBlock pf = luc_plan(fr, lane, s_hist[warp]);
                if (!WRITE) {
                        if (lane == 0)
                                E.dsz[g] = pd.bytes + pf.bytes;
                        return;
                }
                luc_write(o, dl, pd, lane, s_pg[warp]);
                luc_write(o + pd.bytes, fr, pf, lane, s_pg[warp]);
                if (lane == 0 && j < 65535u) {
                        const uint64_t blocksBytes = E.doff[E.dunit_begin[t + 1]] - base; // full blocks + tail
                        uint8_t *      s           = E.index_out + chunk + 14u + blocksBytes + j * kLucSkipEntry;
                        const uint64_t H           = E.hit_begin[d0] - E.hit_begin[tb]; // hits of the term before the block
                        const uint64_t h0          = E.hunit_begin[t];
                        luc_put32(s, uint32_t(14u + (E.doff[g] - base)));                   // indexOffset
                        luc_put32(s + 4, j ? E.docids[d0 - 1] : 0u);                         // lastDocID
                        luc_put32(s + 8, uint32_t(E.hoff[h0 + H / kLucBlock] - E.hoff[h0])); // lastHitsBlockOffset
                        luc_put32(s + 12, uint32_t(j * kLucBlock));                          // totalDocumentsSoFar
                        luc_put32(s + 16, uint32_t(H / kLucBlock * kLucBlock));              // lastHitsBlockTotalHits
                        s[20] = uint8_t(H % kLucBlock), s[21] = 0;                           // curHitsBlockHits
                }
                return;
        }
        // the tail: varbyte(delta) varbyte(freq) per document; its warp also writes the chunk header
        uint32_t len[4], tot{0};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
                len[q] = uint32_t(q) * 32u + uint32_t(lane) < n ? vb_len_of(dl[q]) + vb_len_of(fr[q]) : 0u;
                tot += __reduce_add_sync(0xffffffffu, len[q]);
        }
        if (!WRITE) {
                if (lane == 0)
                        E.dsz[g] = tot;
                return;
        }
        uint32_t run{0};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
                uint32_t a = len[q];
                for (int s = 1; s < 32; s <<= 1) {
                        const uint32_t y = __shfl_up_sync(0xffffffffu, a, s);
                        if (lane >= s)
                                a += y;
                }
                if (len[q])
                        vb_store(vb_store(o + run + a - len[q], dl[q]), fr[q]);
                run += __shfl_sync(0xffffffffu, a, 31);
        }
        if (lane == 0) {
                const uint64_t h0 = E.hunit_begin[t], h1 = E.hunit_begin[t + 1];
                uint8_t *      hd = E.index_out + chunk;
                const uint32_t entries = uint32_t(min(nfull, uint64_t(65535u)));
                luc_put32(hd, uint32_t(E.hoff[h0]));                             // hitsDataOffset
                luc_put32(hd + 4, uint32_t(E.hit_begin[te] - E.hit_begin[tb])); // sumHits
                luc_put32(hd + 8, uint32_t(E.hoff[h1] - E.hoff[h0]));           // positionsChunkSize
                hd[12] = uint8_t(entries), hd[13] = uint8_t(entries >> 8);       // skiplistSize
        }
}

// writes the payload bytes of the lane's hits (val[q] = their sizes) after the ones of the earlier hits of the unit, from o
__device__ __forceinline__ void luc_payload_bytes(uint8_t *o, const EncPayloads &E, uint64_t x0, const uint32_t (&len)[4], int lane) {
        uint32_t run{0};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
                uint32_t a = len[q];
                for (int s = 1; s < 32; s <<= 1) {
                        const uint32_t y = __shfl_up_sync(0xffffffffu, a, s);
                        if (lane >= s)
                                a += y;
                }
                if (len[q]) {
                        const unsigned long long v = E.payloads[x0 + uint32_t(q) * 32u + uint32_t(lane)];
                        uint8_t *                p = o + run + a - len[q];
                        for (uint32_t b = 0; b < len[q]; ++b)
                                p[b] = uint8_t(v >> (8u * b));
                }
                run += __shfl_sync(0xffffffffu, a, 31);
        }
}

// size (WRITE = false) or bytes (WRITE = true) of one hit unit, one warp per unit.  PAYLOADS: every hit carries plens[] / payloads[]
// (positions are given); a position-0 hit is legal when it has a payload.
template <bool WRITE, bool PAYLOADS = false>
__global__ void __launch_bounds__(128) k_enc_lucene_hits(std::conditional_t<PAYLOADS, EncLucenePayloadParams, EncLuceneParams> E) {
        __shared__ uint32_t s_pg[4][kLucPageWords];
        __shared__ uint32_t s_hist[4][33];
        const int           warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const uint64_t      g    = uint64_t(blockIdx.x) * 4u + uint64_t(warp);
        if (g >= E.nhunits)
                return;
        uint32_t t;
        if (!WRITE) {
                t = luc_term_of(E.hunit_begin, E.nterms, g);
                if (lane == 0)
                        E.hterm[g] = t;
        } else
                t = E.hterm[g];
        const uint64_t tb = E.term_begin[t], te = E.term_begin[t + 1];
        const uint64_t hb = E.hit_begin[tb], sum = E.hit_begin[te] - hb;
        const uint64_t j = g - E.hunit_begin[t], nfh = sum / kLucBlock;
        const uint64_t x0 = hb + j * kLucBlock;
        const uint32_t n  = j < nfh ? kLucBlock : uint32_t(sum % kLucBlock);
        uint32_t       val[4], pln[4] = {0u, 0u, 0u, 0u};
        bool           bad = false;
        if (E.positions && n) {
                // the documents of the unit's first and last hits bound every lane's search: the last posting p of the term with
                // hit_begin[p] <= x holds hit x (freq-0 postings share their hit_begin with the next one), x is its first hit iff equal
                auto doc_of = [&](uint64_t x, uint64_t lo, uint64_t hi) {
                        while (lo < hi) {
                                const uint64_t mid = (lo + hi + 1u) >> 1;
                                if (E.hit_begin[mid] <= x)
                                        lo = mid;
                                else
                                        hi = mid - 1u;
                        }
                        return lo;
                };
                const uint64_t pa = doc_of(x0, tb, te - 1u), pb = doc_of(x0 + n - 1u, pa, te - 1u);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                        const uint32_t i = uint32_t(q) * 32u + uint32_t(lane);
                        val[q]           = 0;
                        if (i < n) {
                                const uint64_t x     = x0 + i;
                                const uint64_t p     = doc_of(x, pa, pb);
                                const uint32_t pos   = E.positions[x];
                                const uint32_t prev  = E.hit_begin[p] == x ? 0u : E.positions[x - 1];
                                if constexpr (PAYLOADS) {
                                        pln[q] = E.pay.plens[x];
                                        bad |= (pos == 0u && pln[q] == 0u) || pln[q] > 8u; // lucene_codec.cpp:240-250
                                } else
                                        bad |= pos == 0u;
                                bad |= pos < prev || pos >= (1u << 14); // Limits::MaxPosition (trinity_limits.h:15)
                                val[q] = pos - prev;
                        }
                }
        } else
#pragma unroll
                for (int q = 0; q < 4; ++q)
                        val[q] = uint32_t(q) * 32u + uint32_t(lane) < n ? 1u : 0u; // positions 1..freq: every delta is 1
        if (__any_sync(0xffffffffu, bad)) {
                if (lane == 0) {
                        atomicExch(E.error, 1u);
                        if (!WRITE)
                                E.hsz[g] = 0;
                }
                return;
        }
        uint8_t *o = WRITE ? E.hits_out + E.hoff[g] : nullptr;
        if constexpr (PAYLOADS) {
                if (j < nfh) { // intblock(position deltas) intblock(payload sizes) varbyte(their sum) the payload bytes
                        const LucIntBlock P   = luc_plan(val, lane, s_hist[warp]);
                        const LucIntBlock PL  = luc_plan(pln, lane, s_hist[warp]);
                        const uint32_t    sum = __reduce_add_sync(0xffffffffu, pln[0] + pln[1] + pln[2] + pln[3]);
                        if (!WRITE) {
                                if (lane == 0)
                                        E.hsz[g] = P.bytes + PL.bytes + vb_len_of(sum) + sum;
                                return;
                        }
                        luc_write(o, val, P, lane, s_pg[warp]);
                        luc_write(o + P.bytes, pln, PL, lane, s_pg[warp]);
                        uint8_t *pb = o + P.bytes + PL.bytes + vb_len_of(sum);
                        if (lane == 0)
                                vb_store(o + P.bytes + PL.bytes, sum);
                        luc_payload_bytes(pb, E.pay, x0, pln, lane);
                        return;
                }
                // the tail: varbyte(delta << 1 | changed) [size] per hit, then every payload byte of the tail
                uint32_t len[4], ch[4], tot{0}, ptot{0};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                        const uint32_t i = uint32_t(q) * 32u + uint32_t(lane);
                        ch[q]            = i < n && pln[q] != (i ? uint32_t(E.pay.plens[x0 + i - 1u]) : 0u);
                        len[q]           = i < n ? vb_len_of((val[q] << 1) | ch[q]) + ch[q] : 0u;
                        tot += __reduce_add_sync(0xffffffffu, len[q]);
                        ptot += __reduce_add_sync(0xffffffffu, pln[q]);
                }
                if (!WRITE) {
                        if (lane == 0)
                                E.hsz[g] = tot + ptot;
                        return;
                }
                uint32_t run{0};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                        uint32_t a = len[q];
                        for (int s = 1; s < 32; s <<= 1) {
                                const uint32_t y = __shfl_up_sync(0xffffffffu, a, s);
                                if (lane >= s)
                                        a += y;
                        }
                        if (len[q]) {
                                uint8_t *p = vb_store(o + run + a - len[q], (val[q] << 1) | ch[q]);
                                if (ch[q])
                                        *p = uint8_t(pln[q]);
                        }
                        run += __shfl_sync(0xffffffffu, a, 31);
                }
                luc_payload_bytes(o + tot, E.pay, x0, pln, lane);
        } else {
                if (j < nfh) { // intblock(position deltas), then the payload sizes (all 0: 00 00) and the payload bytes (varbyte(0))
                        const LucIntBlock P = luc_plan(val, lane, s_hist[warp]);
                        if (!WRITE) {
                                if (lane == 0)
                                        E.hsz[g] = P.bytes + 3u;
                                return;
                        }
                        luc_write(o, val, P, lane, s_pg[warp]);
                        if (lane == 0)
                                o[P.bytes] = o[P.bytes + 1] = o[P.bytes + 2] = 0;
                        return;
                }
                // the tail: varbyte(delta << 1) per hit (no payload size change)
                uint32_t len[4], tot{0};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                        len[q] = uint32_t(q) * 32u + uint32_t(lane) < n ? vb_len_of(val[q] << 1) : 0u;
                        tot += __reduce_add_sync(0xffffffffu, len[q]);
                }
                if (!WRITE) {
                        if (lane == 0)
                                E.hsz[g] = tot;
                        return;
                }
                uint32_t run{0};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                        uint32_t a = len[q];
                        for (int s = 1; s < 32; s <<= 1) {
                                const uint32_t y = __shfl_up_sync(0xffffffffu, a, s);
                                if (lane >= s)
                                        a += y;
                        }
                        if (len[q])
                                vb_store(o + run + a - len[q], val[q] << 1);
                        run += __shfl_sync(0xffffffffu, a, 31);
                }
        }
}

// hits before every term: term_hits[t] = hit_begin[term_begin[t]], t <= nterms
__global__ void __launch_bounds__(256) k_enc_lucene_term_hits(const unsigned long long *term_begin, const unsigned long long *hit_begin, uint32_t nterms,
                                                              unsigned long long *term_hits) {
        const uint32_t t = blockIdx.x * 256u + threadIdx.x;
        if (t <= nterms)
                term_hits[t] = hit_begin[term_begin[t]];
}

// chunk offsets (fixed[t]: the headers and skiplists of the terms before t) and hits.data offsets of every term, t <= nterms
__global__ void __launch_bounds__(256) k_enc_lucene_terms(EncLuceneParams E, const unsigned long long *fixed, unsigned long long *term_off,
                                                          unsigned long long *hits_off) {
        const uint32_t t = blockIdx.x * 256u + threadIdx.x;
        if (t > E.nterms)
                return;
        term_off[t] = E.doff[E.dunit_begin[t]] + fixed[t];
        hits_off[t] = E.hoff[E.hunit_begin[t]];
}

cudaError_t launch_enc_lucene_term_hits(const unsigned long long *term_begin, const unsigned long long *hit_begin, uint32_t nterms, unsigned long long *term_hits,
                                        cudaStream_t stream) {
        k_enc_lucene_term_hits<<<nterms / 256u + 1u, 256, 0, stream>>>(term_begin, hit_begin, nterms, term_hits);
        return cudaGetLastError();
}
// pay.plens set: the payload instantiation of the hit units
cudaError_t launch_enc_lucene_sizes(const EncLuceneParams &E, const EncPayloads &pay, cudaStream_t stream) {
        k_enc_lucene_docs<false><<<unsigned((E.ndunits + 3) / 4), 128, 0, stream>>>(E);
        if (pay.plens)
                k_enc_lucene_hits<false, true><<<unsigned((E.nhunits + 3) / 4), 128, 0, stream>>>(EncLucenePayloadParams{E, pay});
        else
                k_enc_lucene_hits<false><<<unsigned((E.nhunits + 3) / 4), 128, 0, stream>>>(E);
        return cudaGetLastError();
}
cudaError_t launch_enc_lucene_terms(const EncLuceneParams &E, const unsigned long long *fixed, unsigned long long *term_off, unsigned long long *hits_off,
                                    cudaStream_t stream) {
        k_enc_lucene_terms<<<E.nterms / 256u + 1u, 256, 0, stream>>>(E, fixed, term_off, hits_off);
        return cudaGetLastError();
}
cudaError_t launch_enc_lucene_write(const EncLuceneParams &E, const EncPayloads &pay, cudaStream_t stream) {
        k_enc_lucene_docs<true><<<unsigned((E.ndunits + 3) / 4), 128, 0, stream>>>(E);
        if (pay.plens)
                k_enc_lucene_hits<true, true><<<unsigned((E.nhunits + 3) / 4), 128, 0, stream>>>(EncLucenePayloadParams{E, pay});
        else
                k_enc_lucene_hits<true><<<unsigned((E.nhunits + 3) / 4), 128, 0, stream>>>(E);
        return cudaGetLastError();
}
