// k_decode_stream_google / k_decode_stream_lucene — whole-list decode (BASELINE.json configs[4]: the postings-decode microbench; also the
// parity probe of the decoders) == PostingsListIterator::next() over whole lists (google_codec.cpp:777-819 + unpack_block :596-639;
// lucene_codec.cpp:568-594 + refill_documents :515-558 + FastPFor<4> __decodeArray fastpfor.h:222-270).  (Included by kernels.cu.)
//
// The first decoders were instruction-bound at a fraction of the HBM roofline: a register-staged copy loop
// (LDG -> STS: the top stall line), a byte-wise varbyte walk through generic pointers and a second pass to find the freq section.
// Here
//   * the bytes of a unit (32 consecutive blocks of one term: a contiguous span of the chunk, positions included) arrive by ONE 1-D bulk
//     copy (cp.async.bulk.shared::cluster.global + mbarrier complete_tx, issued by one lane; SASS UBLKCP / SYNCS), double-buffered per warp:
//     the copy of unit u+1 is in flight while unit u is decoded, and no thread spends an instruction on moving bytes;
//   * GOOGLE: lane = block, every lane walks 32-bit windows of ITS block in shared memory: dense lists take four 1-byte codes per window,
//     sparse lists up to two codes of 1-2 bytes per window (3-5-byte codes on a rare side path), freq sections four codes per window;
//     the freq section starts where the delta walk ends — one pass, no votes (lanes of a unit decode blocks of the same list);
//   * LUCENE: one warp per 128-document block, vertical PFor unpack (lucene_intblock_v), the directory entries of 32 consecutive blocks
//     loaded by the 32 lanes at once.
// Every docID and freq is produced in a register (the checksum variant adds them up, the materialising variant stores them).
#pragma once

// GOOGLE staging buffer = the span of 32 blocks (a template parameter of the kernel: 6 KB for the reference format's 32-document blocks,
// scaled with the block size for the decode sweep; a span that does not fit is read from global memory)
static constexpr uint32_t kDlWarpBytes  = 2 * kSfStage + kSfScratch; // LUCENE: two block buffers + exception scratch

// 64-bit accumulate of a 32-bit value (two instructions; the sums of docIDs exceed 32 bits)
__device__ __forceinline__ void acc64(unsigned long long &s, uint32_t v) {
        s += v;
}

// generic-pointer form of the same walk for spans that do not fit the staging buffer (positions-heavy blocks): straight from global memory
template <bool MAT>
__device__ __forceinline__ void ds_google_block_global(const uint8_t *p, uint32_t n, uint32_t prev, uint32_t last, uint32_t *outd, uint32_t *outf,
                                                       unsigned long long &sumd, unsigned long long &sumf) {
        uint32_t doc = prev;
        for (uint32_t i = 0; i + 1u < n; ++i) {
                doc += varbyte_get(p);
                acc64(sumd, doc);
                if (MAT)
                        outd[i] = doc;
        }
        acc64(sumd, last);
        if (MAT)
                outd[n - 1u] = last;
        for (uint32_t i = 0; i < n; ++i) {
                const uint32_t v = varbyte_get(p);
                sumf += v;
                if (MAT)
                        outf[i] = v;
        }
}

// the freq section of a block: n codes, almost always 1 byte each — four at a time, every lane on its own
template <bool MAT>
__device__ __forceinline__ void ds_google_freqs(uint32_t sp, uint32_t n, uint32_t *outf, unsigned long long &sumf) {
        uint32_t i = 0;
        while (i < n) {
                const uint32_t a = sp & ~3u;
                const uint32_t w = __funnelshift_r(lds_u32(a), lds_u32(a + 4u), (sp & 3u) * 8u);
                if ((w & 0x80808080u) == 0u && i + 4u <= n && (!MAT || (i & 3u) == 0u)) {
                        sumf += __dp4a(w, 0x01010101u, 0u);
                        if (MAT)
                                *reinterpret_cast<uint4 *>(outf + i) = make_uint4(w & 0xffu, __byte_perm(w, 0u, 0x4441u), __byte_perm(w, 0u, 0x4442u), w >> 24);
                        sp += 4u;
                        i += 4u;
                } else {
                        const uint32_t b0 = w & 0xffu;
                        uint32_t       v, len;
                        if (b0 < 0xc0u) {
                                const uint32_t two = b0 >> 7;
                                v   = two ? (((b0 & 0x3fu) << 8) | __byte_perm(w, 0u, 0x4441u)) : b0;
                                len = 1u + two;
                        } else if (b0 < 0xe0u) {
                                v   = ((b0 & 0x1fu) << 16) | ((w >> 8) & 0xffffu);
                                len = 3u;
                        } else if (b0 < 0xf0u) {
                                v   = ((b0 & 0x0fu) << 24) | (((w >> 8) & 0xffu) << 16) | (((w >> 16) & 0xffu) << 8) | (w >> 24);
                                len = 4u;
                        } else {
                                const uint32_t a1 = (sp + 1u) & ~3u;
                                v   = __funnelshift_r(lds_u32(a1), lds_u32(a1 + 4u), ((sp + 1u) & 3u) * 8u);
                                len = 5u;
                        }
                        sumf += v;
                        if (MAT)
                                outf[i] = v;
                        sp += len;
                        ++i;
                }
        }
}

// SPARSE lists (average gap >= 48: most doc deltas are 2-byte codes, so the warp-voted 4-wide step above would fail on almost every
// window): every lane walks ITS block on its own — no votes — taking up to TWO codes of 1-2 bytes out of each 32-bit window (two such
// codes always fit), a rare side path for 3-5-byte codes; the freq section (1-byte codes) goes four at a time.
template <bool MAT>
__device__ __forceinline__ void ds_google_block_sparse(uint32_t sp, uint32_t n, uint32_t prev, uint32_t last, uint32_t *outd, uint32_t *outf, unsigned long long &sumd,
                                                       unsigned long long &sumf) {
        const uint32_t nd  = n - 1u;
        uint32_t       doc = prev, i = 0;
        uint4          rowbuf = make_uint4(0, 0, 0, 0);
        auto           put    = [&](uint32_t at, uint32_t v) { // four docIDs per 16-byte store
                const uint32_t s4 = at & 3u;
                if (s4 == 0u) rowbuf.x = v;
                else if (s4 == 1u) rowbuf.y = v;
                else if (s4 == 2u) rowbuf.z = v;
                else {
                        rowbuf.w = v;
                        *reinterpret_cast<uint4 *>(outd + (at & ~3u)) = rowbuf;
                }
        };
        while (i < nd) {
                const uint32_t a  = sp & ~3u;
                const uint32_t w  = __funnelshift_r(lds_u32(a), lds_u32(a + 4u), (sp & 3u) * 8u); // bytes sp .. sp+3
                const uint32_t b0 = w & 0xffu;
                if (b0 >= 0xc0u) { // 3..5-byte code
                        uint32_t v, len;
                        if (b0 < 0xe0u) {
                                v   = ((b0 & 0x1fu) << 16) | ((w >> 8) & 0xffffu);
                                len = 3u;
                        } else if (b0 < 0xf0u) {
                                v   = ((b0 & 0x0fu) << 24) | (((w >> 8) & 0xffu) << 16) | (((w >> 16) & 0xffu) << 8) | (w >> 24);
                                len = 4u;
                        } else {
                                const uint32_t a1 = (sp + 1u) & ~3u;
                                v   = __funnelshift_r(lds_u32(a1), lds_u32(a1 + 4u), ((sp + 1u) & 3u) * 8u);
                                len = 5u;
                        }
                        doc += v;
                        sumd += doc;
                        if (MAT)
                                put(i, doc);
                        sp += len;
                        ++i;
                        continue;
                }
                const uint32_t two = b0 >> 7;
                uint32_t       len = 1u + two;
                doc += two ? (((b0 & 0x3fu) << 8) | __byte_perm(w, 0u, 0x4441u)) : b0;
                sumd += doc;
                if (MAT)
                        put(i, doc);
                ++i;
                // the second code of the window
                const uint32_t w2 = w >> (8u * len), c0 = w2 & 0xffu;
                if (i < nd && c0 < 0xc0u) {
                        const uint32_t two2 = c0 >> 7;
                        doc += two2 ? (((c0 & 0x3fu) << 8) | ((w2 >> 8) & 0xffu)) : c0;
                        sumd += doc;
                        if (MAT)
                                put(i, doc);
                        ++i;
                        len += 1u + two2;
                }
                sp += len;
        }
        sumd += last;
        if (MAT) {
                const uint32_t s4 = nd & 3u, base = nd & ~3u;
                if (s4 == 0u) outd[base] = last;
                else if (s4 == 1u) { outd[base] = rowbuf.x; outd[base + 1] = last; }
                else if (s4 == 2u) { outd[base] = rowbuf.x; outd[base + 1] = rowbuf.y; outd[base + 2] = last; }
                else *reinterpret_cast<uint4 *>(outd + base) = make_uint4(rowbuf.x, rowbuf.y, rowbuf.z, last);
        }
        ds_google_freqs<MAT>(sp, n, outf, sumf);
}

// DENSE lists without votes: every lane on its own takes four 1-byte codes per window when it can, else one code (1-2 bytes branch-free,
// longer ones on a side path).  Lanes of a unit decode blocks of the same list, so they agree almost always; when one lane meets a longer
// code the others idle for that step instead of the whole warp paying two votes on every step.
template <bool MAT>
__device__ __forceinline__ void ds_google_block_dense(uint32_t sp, uint32_t n, uint32_t prev, uint32_t last, uint32_t *outd, uint32_t *outf, unsigned long long &sumd,
                                                      unsigned long long &sumf) {
        const uint32_t nd  = n - 1u;
        uint32_t       doc = prev, i = 0;
        uint4          rowbuf = make_uint4(0, 0, 0, 0);
        while (i < nd) {
                const uint32_t a = sp & ~3u;
                const uint32_t w = __funnelshift_r(lds_u32(a), lds_u32(a + 4u), (sp & 3u) * 8u); // bytes sp .. sp+3
                if ((w & 0x80808080u) == 0u && i + 4u <= nd && (!MAT || (i & 3u) == 0u)) {
                        const uint32_t d0 = doc + (w & 0xffu), d1 = d0 + __byte_perm(w, 0u, 0x4441u), d2 = d1 + __byte_perm(w, 0u, 0x4442u), d3 = d2 + (w >> 24);
                        doc = d3;
                        sumd += static_cast<unsigned long long>(d0) + d1 + d2 + d3;
                        if (MAT)
                                *reinterpret_cast<uint4 *>(outd + i) = make_uint4(d0, d1, d2, d3);
                        sp += 4u;
                        i += 4u;
                        continue;
                }
                const uint32_t b0 = w & 0xffu;
                uint32_t       v, len;
                if (b0 < 0xc0u) {
                        const uint32_t two = b0 >> 7;
                        v   = two ? (((b0 & 0x3fu) << 8) | __byte_perm(w, 0u, 0x4441u)) : b0;
                        len = 1u + two;
                } else if (b0 < 0xe0u) {
                        v   = ((b0 & 0x1fu) << 16) | ((w >> 8) & 0xffffu);
                        len = 3u;
                } else if (b0 < 0xf0u) {
                        v   = ((b0 & 0x0fu) << 24) | (((w >> 8) & 0xffu) << 16) | (((w >> 16) & 0xffu) << 8) | (w >> 24);
                        len = 4u;
                } else {
                        const uint32_t a1 = (sp + 1u) & ~3u;
                        v   = __funnelshift_r(lds_u32(a1), lds_u32(a1 + 4u), ((sp + 1u) & 3u) * 8u);
                        len = 5u;
                }
                doc += v;
                sumd += doc;
                if (MAT) {
                        const uint32_t s4 = i & 3u;
                        if (s4 == 0u) rowbuf.x = doc;
                        else if (s4 == 1u) rowbuf.y = doc;
                        else if (s4 == 2u) rowbuf.z = doc;
                        else {
                                rowbuf.w = doc;
                                *reinterpret_cast<uint4 *>(outd + (i & ~3u)) = rowbuf;
                        }
                }
                sp += len;
                ++i;
        }
        sumd += last;
        if (MAT) {
                const uint32_t s4 = nd & 3u, base = nd & ~3u;
                if (s4 == 0u) outd[base] = last;
                else if (s4 == 1u) { outd[base] = rowbuf.x; outd[base + 1] = last; }
                else if (s4 == 2u) { outd[base] = rowbuf.x; outd[base + 1] = rowbuf.y; outd[base + 2] = last; }
                else *reinterpret_cast<uint4 *>(outd + base) = make_uint4(rowbuf.x, rowbuf.y, rowbuf.z, last);
        }
        ds_google_freqs<MAT>(sp, n, outf, sumf);
}

// unit = 32 consecutive blocks of one term, one warp per unit, units handed out with a fixed stride.  The host lays the units out
// (DecUnit); the kernel is a three-stage software pipeline per warp: unit descriptor (u+3) -> directory entries (u+2) -> bulk copy of
// the span (u+1) -> decode (u).  Loaded values stay RAW in registers until the stage that needs them (no select behind a load: a select
// right after its load is a stall on that load), so no load sits on the critical path of a decode.
template <bool MAT, uint32_t kDsStage>
__global__ void __launch_bounds__(kThreads) k_decode_stream_google(DevIndex ix, const DecUnit *units, const uint64_t *out_base, uint32_t total_units, uint32_t *docids,
                                                                  uint32_t *freqs, unsigned long long *sums) {
        __shared__ __align__(8) unsigned long long s_bar[kWarps * 2];
        const int      lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        uint8_t *      stage   = dyn_smem + size_t(warp) * (2 * kDsStage);
        const uint32_t stage_s = uint32_t(__cvta_generic_to_shared(stage));
        const uint32_t bar_s   = uint32_t(__cvta_generic_to_shared(&s_bar[warp * 2]));
        if (lane == 0) {
                mbar_init(bar_s, 1);
                mbar_init(bar_s + 8, 1);
                asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
        const uint32_t stride = gridDim.x * kWarps;
        const uint32_t bd     = ix.block_docs;
        const uint32_t lastU  = total_units - 1u; // (the host launches no empty grid)

        struct Desc { // raw descriptor words of a unit (clamped to the last unit past the end; `valid` says which)
                uint4 x;
                uint2 y;
                bool  valid;
        };
        struct Dir { // this lane's raw directory words of a unit
                uint32_t off, offn, last, prevRaw;
                Desc     d;
        };
        auto load_desc = [&](uint32_t u) {
                Desc D;
                D.valid            = u < total_units;
                const DecUnit *pu  = units + min(u, lastU);
                D.x                = __ldg(reinterpret_cast<const uint4 *>(pu));
                D.y                = __ldg(reinterpret_cast<const uint2 *>(pu) + 2);
                return D;
        };
        auto load_dir = [&](const Desc &D) { // D was loaded an iteration ago; every lane loads (lanes past the unit re-read its last block)
                Dir            R;
                const uint32_t cnt = D.x.y; // >= 1 for every descriptor the host writes
                const uint32_t e   = D.x.x + min(uint32_t(lane), cnt - 1u);
                R.off     = __ldg(ix.blk_off + e);
                R.offn    = __ldg(ix.blk_off + e + 1u);
                R.last    = __ldg(ix.blk_last + e);
                R.prevRaw = __ldg(ix.blk_last + max(e, 1u) - 1u);
                R.d       = D;
                return R;
        };
        uint32_t seq_issue = 0, seq_wait = 0;
        // the span of a unit: [first_off, end) with a 16-byte aligned window around it.  Computed (two shuffles of loaded directory words)
        // at the END of an iteration for the unit after the next one — a whole decode after its loads were issued — and carried in registers.
        struct Span {
                uint32_t abase, bytes;
                bool     staged; // it goes through the staging buffer (else the lanes read global memory)
        };
        auto span_of = [&](const Dir &R) {
                Span           S;
                const uint32_t cnt       = R.d.x.y;
                const uint32_t first_off = __shfl_sync(0xffffffffu, R.off, 0);
                const uint32_t end       = __shfl_sync(0xffffffffu, R.offn, int(cnt) - 1);
                S.abase                  = first_off & ~15u;
                S.bytes                  = ((end + 15u) & ~15u) - S.abase;
                S.staged                 = R.d.valid && S.bytes <= kDsStage;
                return S;
        };
        auto issue = [&](const Span &S) {
                if (S.staged) {
                        if (lane == 0) {
                                const uint32_t bsel = seq_issue & 1u;
                                mbar_expect_tx(bar_s + bsel * 8u, S.bytes);
                                bulk_g2s(stage_s + bsel * kDsStage, ix.index + S.abase, S.bytes, bar_s + bsel * 8u);
                        }
                        ++seq_issue;
                }
        };

        uint32_t unit = blockIdx.x * kWarps + warp;
        Dir      cur  = load_dir(load_desc(unit));
        Dir      nxt  = load_dir(load_desc(unit + stride));
        Desc     d2   = load_desc(unit + 2u * stride);
        Span     scur = span_of(cur), snxt = span_of(nxt);
        issue(scur);
        // checksums are kept per warp across the units of one term (units of a term are mostly handled in a row by the same warps) and
        // flushed when the term changes
        unsigned long long accd = 0, accf = 0;
        uint32_t           accti = 0xffffffffu;
        auto               flush = [&]() {
                for (int d = 16; d > 0; d >>= 1) {
                        accd += __shfl_xor_sync(0xffffffffu, accd, d);
                        accf += __shfl_xor_sync(0xffffffffu, accf, d);
                }
                if (lane == 0 && sums && accti != 0xffffffffu) {
                        atomicAdd(&sums[2 * accti], accd);
                        atomicAdd(&sums[2 * accti + 1], accf);
                }
                accd = accf = 0;
        };
        for (; unit < total_units; unit += stride) {
                issue(snxt);
                const Dir  nn = load_dir(d2);                    // directory loads of u+2: in flight while u is decoded
                const Desc d3 = load_desc(unit + 3u * stride);
                const uint32_t abase  = scur.abase;
                const bool     staged = scur.staged;
                uint32_t       bsel   = 0;
                if (staged) {
                        bsel = seq_wait & 1u;
                        mbar_wait(bar_s + bsel * 8u, (seq_wait >> 1) & 1u);
                        ++seq_wait;
                }
                const uint32_t cnt = cur.d.x.y, ti = cur.d.y.x, g0 = cur.d.y.y, lastN = cur.d.x.w;
                if (ti != accti) {
                        flush();
                        accti = ti;
                }
                const bool     active = uint32_t(lane) < cnt;
                const uint32_t prev   = (cur.d.x.z && lane == 0) ? 0u : cur.prevRaw;
                const uint32_t n      = (lastN && uint32_t(lane) + 1u == cnt) ? lastN : bd;
                // dense or sparse walk: decided per unit from its docID span (uniform across the warp)
                const uint32_t lastDoc = __shfl_sync(0xffffffffu, cur.last, int(cnt) - 1), firstPrev = __shfl_sync(0xffffffffu, prev, 0);
                const bool     dense   = (lastDoc - firstPrev) < 48u * cnt * bd;
                if (active) {
                        const size_t row = MAT ? size_t(out_base[ti]) + (size_t(g0) + size_t(lane)) * bd : 0;
                        uint32_t *   od  = MAT ? docids + row : nullptr;
                        uint32_t *   of  = MAT ? freqs + row : nullptr;
                        if (!staged)
                                ds_google_block_global<MAT>(ix.index + cur.off, n, prev, cur.last, od, of, accd, accf);
                        else if (dense)
                                ds_google_block_dense<MAT>(stage_s + bsel * kDsStage + (cur.off - abase), n, prev, cur.last, od, of, accd, accf);
                        else
                                ds_google_block_sparse<MAT>(stage_s + bsel * kDsStage + (cur.off - abase), n, prev, cur.last, od, of, accd, accf);
                }
                __syncwarp();
                cur  = nxt;
                nxt  = nn;
                d2   = d3;
                scur = snxt;
                snxt = span_of(nn); // (its loads are a whole decode old)
        }
        flush();
}

// unit = 32 consecutive blocks of one term (lane j loads the directory entries of block j), the warp decodes them one after the other
template <bool MAT>
__global__ void __launch_bounds__(kThreads) k_decode_stream_lucene(DevIndex ix, const DecUnit *units, const uint64_t *out_base, uint32_t total_units, uint32_t *docids,
                                                                  uint32_t *freqs, unsigned long long *sums) {
        __shared__ __align__(8) unsigned long long s_bar[kWarps * 2];
        const int      lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        uint8_t *      stage   = dyn_smem + size_t(warp) * kDlWarpBytes;
        uint32_t *     scratch = reinterpret_cast<uint32_t *>(stage + 2 * kSfStage);
        const uint32_t stage_s = uint32_t(__cvta_generic_to_shared(stage));
        const uint32_t bar_s   = uint32_t(__cvta_generic_to_shared(&s_bar[warp * 2]));
        if (lane == 0) {
                mbar_init(bar_s, 1);
                mbar_init(bar_s + 8, 1);
                asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
        uint32_t seq_issue = 0, seq_wait = 0;
        for (uint32_t unit = blockIdx.x * kWarps + warp; unit < total_units; unit += gridDim.x * kWarps) {
                const uint4    dx   = __ldg(reinterpret_cast<const uint4 *>(units + unit));
                const uint2    dy   = __ldg(reinterpret_cast<const uint2 *>(units + unit) + 2);
                const uint32_t tcur = dy.x, g0 = dy.y, ucnt = dx.y, tailDocs = dx.w; // tailDocs: documents of the unit's last block if that is the term's tail block
                const bool     have = uint32_t(lane) < ucnt;
                uint32_t       off = 0, offn = 0, prev = 0;
                if (have) {
                        const uint32_t e = dx.x + uint32_t(lane);
                        off  = __ldg(ix.blk_off + e);
                        offn = __ldg(ix.blk_off + e + 1u);
                        prev = (dx.z && lane == 0) ? 0u : __ldg(ix.blk_last + e - 1u);
                }
                const uint32_t nblk = __popc(__ballot_sync(0xffffffffu, have));
                auto           issue = [&](uint32_t j) {
                        const uint32_t o = __shfl_sync(0xffffffffu, off, int(j)), on = __shfl_sync(0xffffffffu, offn, int(j));
                        const uint32_t abase = o & ~15u, bytes = min(((on + 15u) & ~15u) - abase, kSfStage);
                        if (lane == 0) {
                                const uint32_t bsel = seq_issue & 1u;
                                mbar_expect_tx(bar_s + bsel * 8u, bytes);
                                bulk_g2s(stage_s + bsel * kSfStage, ix.index + abase, bytes, bar_s + bsel * 8u);
                        }
                        ++seq_issue;
                };
                unsigned long long sumd = 0, sumf = 0;
                const size_t       trow = MAT ? size_t(out_base[tcur]) : 0;
                if (nblk)
                        issue(0);
                for (uint32_t j = 0; j < nblk; ++j) {
                        if (j + 1u < nblk)
                                issue(j + 1u);
                        const uint32_t bsel = seq_wait & 1u;
                        mbar_wait(bar_s + bsel * 8u, (seq_wait >> 1) & 1u);
                        ++seq_wait;
                        const uint8_t *s    = stage + bsel * kSfStage;
                        const uint32_t oj   = __shfl_sync(0xffffffffu, off, int(j));
                        const uint32_t pj   = __shfl_sync(0xffffffffu, prev, int(j));
                        const uint32_t bj   = g0 + j;
                        const uint32_t skew = oj & 15u;
                        uint32_t *     od   = MAT ? docids + trow + size_t(bj) * 128u : nullptr;
                        uint32_t *     of   = MAT ? freqs + trow + size_t(bj) * 128u : nullptr;
                        if (!(tailDocs && j + 1u == nblk)) {
                                uint32_t d[4], fr[4], dbits, fbits;
                                const uint32_t o2 = lucene_intblock_v(s, skew, lane, d, scratch, dbits);
                                (void)lucene_intblock_v(s, o2, lane, fr, scratch, fbits);
                                uint32_t base = pj;
#pragma unroll
                                for (int g = 0; g < 4; ++g) {
                                        const uint32_t sc = warp_incl_scan(d[g], lane);
                                        d[g]              = base + sc;
                                        base += __shfl_sync(0xffffffffu, sc, 31);
                                        sumd += d[g];
                                        sumf += fr[g];
                                        if (MAT) { // value l + 32 g: consecutive lanes store consecutive words
                                                od[lane + 32 * g] = d[g];
                                                of[lane + 32 * g] = fr[g];
                                        }
                                }
                        } else if (lane == 0) { // tail block: (varbyte delta, varbyte freq) pairs (lucene_codec.cpp:527-550)
                                const uint8_t *pp   = s + skew;
                                uint32_t       doc  = pj;
                                for (uint32_t i = 0; i < tailDocs; ++i) {
                                        doc += varbyte_get(pp);
                                        const uint32_t f = varbyte_get(pp);
                                        sumd += doc;
                                        sumf += f;
                                        if (MAT) {
                                                od[i] = doc;
                                                of[i] = f;
                                        }
                                }
                        }
                        __syncwarp();
                }
                for (int d = 16; d > 0; d >>= 1) {
                        sumd += __shfl_xor_sync(0xffffffffu, sumd, d);
                        sumf += __shfl_xor_sync(0xffffffffu, sumf, d);
                }
                if (lane == 0 && sums && nblk) {
                        atomicAdd(&sums[2 * tcur], sumd);
                        atomicAdd(&sums[2 * tcur + 1], sumf);
                }
                __syncwarp();
        }
}

template <uint32_t STAGE> static const void *decode_google_fn(bool mat) {
        return mat ? (const void *)k_decode_stream_google<true, STAGE> : (const void *)k_decode_stream_google<false, STAGE>;
}

cudaError_t launch_decode_stream(const DevIndex &ix, const DecUnit *units, const uint64_t *out_base, uint32_t total_units, uint32_t *docids, uint32_t *freqs,
                                 unsigned long long *sums, int num_sms, cudaStream_t stream) {
        const bool  mat = docids != nullptr;
        size_t      smem;
        const void *fn;
        if (ix.codec == 0) { // staging sized for the span of 32 blocks of block_docs documents (~4.6 bytes per posting with positions)
                const uint32_t bd = ix.block_docs;
                if (bd <= 16) {
                        fn   = decode_google_fn<3072>(mat);
                        smem = size_t(kWarps) * 2 * 3072;
                } else if (bd <= 32) {
                        fn   = decode_google_fn<6144>(mat);
                        smem = size_t(kWarps) * 2 * 6144;
                } else if (bd <= 64) {
                        fn   = decode_google_fn<12288>(mat);
                        smem = size_t(kWarps) * 2 * 12288;
                } else {
                        fn   = decode_google_fn<24576>(mat);
                        smem = size_t(kWarps) * 2 * 24576;
                }
        } else {
                fn   = mat ? (const void *)k_decode_stream_lucene<true> : (const void *)k_decode_stream_lucene<false>;
                smem = size_t(kWarps) * kDlWarpBytes;
        }
        cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
        if (e != cudaSuccess)
                return e;
        int per = 0;
        e       = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, fn, kThreads, smem);
        if (e != cudaSuccess)
                return e;
        const int grid = int(std::min<uint64_t>(uint64_t(num_sms) * std::max(per, 1), (uint64_t(total_units) + kWarps - 1) / kWarps));
        void *args[] = {(void *)&ix, (void *)&units, (void *)&out_base, (void *)&total_units, (void *)&docids, (void *)&freqs, (void *)&sums};
        return cudaLaunchKernel(fn, dim3(grid), dim3(kThreads), args, smem, stream);
}
