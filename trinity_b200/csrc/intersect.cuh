// Query-token intersections (trn_intersect == Trinity::intersect_impl, intersect.cpp:5-170).  (Included by kernels.cu.)
//
// The reference walks the union of all the tokens' posting lists in docID order and feeds the mask of every considered document (the
// groups it holds; not the whole query's mask, not a masked document) to a sequential state machine (ctx::consider).  That machine is
// restated exactly (DESIGN.md §4, isectplan.h) so that every document is handled on its own:
//   pass A (k_isect_masks)  every distinct mask with its first docID, and the mask of each tile's last considered document;
//   host  (isect_plan)      the epochs (stretches between two pushes of the antichain) and their arrays, from those masks alone;
//   pass B (k_isect_count)  per considered document: its epoch, its target in that epoch's array, whether it starts a run of equal
//                           masks (its considered neighbour, or the carry from earlier tiles) -> +1 / +0 on the target's final count.
// Both passes run one WARP per (request, docID tile) work item, like k_exec_docs: the warp decodes every token of the request that
// touches the tile into its group's bitmap with the step-program leaf decoders (google_leaf_warp / lucene_leaf_warp; resident bitmaps
// of dense GOOGLE terms are ORed in instead), then walks the tile 32 documents at a time with lane = document.
#pragma once

static constexpr int      kIsectWarps    = 4;
static constexpr uint32_t kIsectSlotBits = 16; // a warp's group bitmaps hold 2^16 bits: tile = 2^16 / max(8, groups rounded up to a power of two)
static constexpr uint32_t kIsectWarpBytes = (1u << kIsectSlotBits) / 8u + kDocsStageBytes1;

// the tile's group bitmaps: group g in slots[g * NW ..), masked documents not removed yet
template <bool LUC>
__device__ void isect_build(const IsectParams &P, const IsectReq &R, uint32_t lo, uint32_t W, uint32_t NW, uint32_t *slots, uint8_t *stage, int lane,
                            uint32_t bar_s, uint32_t &seq) {
        {
                uint4 *        s4 = reinterpret_cast<uint4 *>(slots);
                const uint32_t n4 = R.ngroups * (NW >> 2);
                for (uint32_t i = lane; i < n4; i += 32)
                        s4[i] = make_uint4(0, 0, 0, 0);
        }
        __syncwarp();
        for (uint32_t k = 0; k < R.ntok; ++k) {
                const uint2   tg = P.tok[R.tok_begin + k];
                const DevTerm T  = P.ix.terms[tg.x];
                if (!T.nblocks || lo > T.last_doc || lo + (W - 1u) < T.first_doc)
                        continue;
                uint32_t *dst = slots + size_t(tg.y) * NW;
                if constexpr (!LUC) {
                        if (P.ix.dense_off) {
                                const uint32_t o = __ldg(P.ix.dense_off + tg.x);
                                if (o != kDenseNone) { // the tile lies inside the bitmap's span
                                        const uint4 *s4 = reinterpret_cast<const uint4 *>(P.ix.dense + o + ((lo - ((T.first_doc >> kDenseAlignShift) << kDenseAlignShift)) >> 5));
                                        uint4 *      d4 = reinterpret_cast<uint4 *>(dst);
                                        for (uint32_t i = lane; i < (NW >> 2); i += 32) {
                                                const uint4 a = d4[i], b = __ldg(s4 + i);
                                                d4[i]         = make_uint4(a.x | b.x, a.y | b.y, a.z | b.z, a.w | b.w);
                                        }
                                        __syncwarp();
                                        continue;
                                }
                        }
                }
                uint32_t bA, bB;
                tile_block_range(P.ix, T, lo, W, bA, bB);
                if (bA > bB)
                        continue;
                BitSink bs;
                bs.init(dst, nullptr, M_OR);
                if constexpr (!LUC)
                        google_leaf_warp(P.ix, T, bA, bB, lo, lo + W, bs, nullptr, stage, kDocsStageBytes1, lane);
                else
                        lucene_leaf_warp(P.ix, T, bA, bB, lo, lo + W, bs, nullptr, stage, lane, bar_s, seq);
                __syncwarp();
        }
}

// lane = document lo + 32 w + lane: the groups it holds
__device__ __forceinline__ uint64_t isect_doc_mask(const uint32_t *slots, uint32_t G, uint32_t NW, uint32_t w, int lane) {
        uint64_t m = 0;
        for (uint32_t g = 0; g < G; ++g)
                m |= uint64_t((slots[g * NW + w] >> lane) & 1u) << g;
        return m;
}

__device__ __forceinline__ uint64_t isect_hash(uint64_t x) { // splitmix64's finalizer
        x ^= x >> 30;
        x *= 0xbf58476d1ce4e5b9ull;
        x ^= x >> 27;
        x *= 0x94d049bb133111ebull;
        return x ^ (x >> 31);
}

// distinct mask m seen at docID doc: insert it into request r's table, keep the smallest docID
__device__ void isect_insert(const IsectParams &P, uint32_t r, const IsectReq &R, uint64_t m, uint32_t doc) {
        if (*reinterpret_cast<volatile uint32_t *>(P.ndist + r) > P.max_masks)
                return; // the request is refused anyway (TRN_ERR_CAPACITY)
        unsigned long long *K   = P.keys + R.table_base;
        uint32_t *          F   = P.first + R.table_base;
        const uint64_t      msk = R.slots - 1u;
        uint64_t            h   = isect_hash(m) & msk;
        for (uint64_t p = 0; p < R.slots; ++p, h = (h + 1u) & msk) {
                unsigned long long k = *reinterpret_cast<volatile unsigned long long *>(K + h);
                if (k == 0ull) {
                        k = atomicCAS(K + h, 0ull, (unsigned long long)m);
                        if (k == 0ull) {
                                atomicAdd(P.ndist + r, 1u);
                                k = m;
                        }
                }
                if (k == m) {
                        atomicMin(F + h, doc);
                        return;
                }
        }
        atomicExch(P.error, 1u);
}

// the work item's request and tile; false when the tickets are used up
__device__ __forceinline__ bool isect_ticket(const IsectParams &P, uint32_t &item, uint32_t &r, int lane) {
        uint32_t t = 0;
        if (lane == 0)
                t = atomicAdd(P.ticket, 1u);
        item = __shfl_sync(0xffffffffu, t, 0);
        if (item >= P.total_items)
                return false;
        uint32_t a = 0, b = P.nreq;
        while (b - a > 1u) {
                const uint32_t mid = (a + b) >> 1;
                if (P.reqs[mid].item_base <= item) a = mid;
                else b = mid;
        }
        r = a;
        return true;
}

// PASS B == false: pass A (distinct masks, tile_last); PASS B == true: the counts
template <bool LUC, bool PASSB> __global__ void __launch_bounds__(kIsectWarps * 32) k_isect(IsectParams P) {
        __shared__ __align__(8) unsigned long long s_lbar[kIsectWarps]; // LUCENE: one mbarrier per warp for its block copies
        uint32_t lseq = 0;
        if constexpr (LUC) {
                if ((threadIdx.x & 31) == 0) {
                        mbar_init(uint32_t(__cvta_generic_to_shared(&s_lbar[threadIdx.x >> 5])), 1);
                        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
                }
                __syncthreads();
        }
        const int      lane  = threadIdx.x & 31, warp = threadIdx.x >> 5;
        uint32_t *     slots = reinterpret_cast<uint32_t *>(dyn_smem + size_t(kIsectWarpBytes) * warp);
        uint8_t *      stage = dyn_smem + size_t(kIsectWarpBytes) * warp + ((1u << kIsectSlotBits) / 8u);
        const uint32_t bar_s = uint32_t(__cvta_generic_to_shared(&s_lbar[warp]));
        uint32_t       item, r;
        while (isect_ticket(P, item, r, lane)) {
                const IsectReq R    = P.reqs[r];
                const uint32_t tile = R.tile_lo + (item - R.item_base);
                const uint32_t W = 1u << R.shift, NW = W >> 5, lo = tile << R.shift;
                isect_build<LUC>(P, R, lo, W, NW, slots, stage, lane, bar_s, lseq);
                uint64_t       last = PASSB ? P.carry[item] : 0ull; // the mask of the last considered document so far (pass B: from earlier tiles on)
                const uint32_t ne   = R.nepochs;
                for (uint32_t w = 0; w < NW; ++w) {
                        const uint64_t m    = isect_doc_mask(slots, R.ngroups, NW, w, lane);
                        const uint32_t doc  = lo + 32u * w + uint32_t(lane);
                        const bool     mkd  = P.ix.masked && ((P.ix.masked[(lo >> 5) + w] >> lane) & 1u);
                        const bool     cons = m != 0ull && m != R.orig_mask && !mkd;
                        const unsigned cb   = __ballot_sync(0xffffffffu, cons);
                        if (!cb)
                                continue;
                        if constexpr (!PASSB) {
                                // one insert per distinct mask of the 32 documents, by its first (lowest) lane
                                const unsigned grp = __match_any_sync(0xffffffffu, cons ? m : 0ull);
                                if (cons && !(grp & ((1u << lane) - 1u)))
                                        isect_insert(P, r, R, m, doc);
                        } else {
                                const unsigned below = cb & ((1u << lane) - 1u);
                                const uint64_t nb    = __shfl_sync(0xffffffffu, m, below ? 31 - __clz(int(below)) : lane);
                                const uint64_t prev  = below ? nb : last; // the previous considered document's mask
                                int32_t        slot  = -1;
                                if (cons) {
                                        uint32_t a = 0, b = ne; // the epoch: the last one starting at or before doc
                                        while (b - a > 1u) {
                                                const uint32_t mid = (a + b) >> 1;
                                                if (P.epoch_start[R.epoch_begin + mid] <= doc) a = mid;
                                                else b = mid;
                                        }
                                        const uint32_t s0 = P.epoch_off[R.epoch_begin + a], s1 = P.epoch_off[R.epoch_begin + a + 1u];
                                        uint32_t       i  = s0;
                                        while (i < s1 && (P.snap_mask[i] & m) != m)
                                                ++i;
                                        if (i == s1)
                                                atomicExch(P.error, 1u);
                                        else if (prev == m) // a run goes on: ctx::consider adds to matches[indexPrev], a uint8_t index
                                                slot = P.snap_slot[s0 + ((i - s0) & 255u)];
                                        else if (P.snap_mask[i] == m) // a run starts on its own entry (absorbed by a strict superset: not counted)
                                                slot = P.snap_slot[i];
                                }
                                const unsigned grp = __match_any_sync(0xffffffffu, slot);
                                if (slot >= 0 && !(grp & ((1u << lane) - 1u)))
                                        atomicAdd(P.counts + slot, uint32_t(__popc(grp)));
                        }
                        last = __shfl_sync(0xffffffffu, m, 31 - __clz(int(cb)));
                }
                if (!PASSB && lane == 0)
                        P.tile_last[item] = last;
                __syncwarp(); // every lane is done with the bitmaps before the next tile clears them
        }
}

// the distinct masks of every request, densely: request r's at out[base[r] ..), in no particular order
__global__ void k_isect_compact(IsectParams P, uint64_t total_slots, const uint64_t *base, uint32_t *cursor, unsigned long long *out_mask, uint32_t *out_first) {
        for (uint64_t s = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; s < total_slots; s += uint64_t(gridDim.x) * blockDim.x) {
                const unsigned long long k = P.keys[s];
                if (!k)
                        continue;
                uint32_t a = 0, b = P.nreq;
                while (b - a > 1u) {
                        const uint32_t mid = (a + b) >> 1;
                        if (P.reqs[mid].table_base <= s) a = mid;
                        else b = mid;
                }
                const uint32_t pos = atomicAdd(cursor + a, 1u);
                if (pos < P.ndist[a]) {
                        out_mask[base[a] + pos]  = k;
                        out_first[base[a] + pos] = P.first[s];
                }
        }
}

// carry[item] = the mask of the last considered document of the request's tiles before the item's (0: none); one warp per request
__global__ void k_isect_carry(IsectParams P, unsigned long long *carry) {
        const uint32_t r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
        const int      lane = threadIdx.x & 31;
        if (r >= P.nreq)
                return;
        const IsectReq R = P.reqs[r];
        uint64_t       c = 0;
        for (uint32_t t0 = 0; t0 < R.ntiles; t0 += 32u) {
                const uint32_t t   = t0 + uint32_t(lane);
                const uint64_t v   = t < R.ntiles ? P.tile_last[R.item_base + t] : 0ull;
                const unsigned nz  = __ballot_sync(0xffffffffu, v != 0ull);
                const unsigned bel = nz & ((1u << lane) - 1u);
                const uint64_t nb  = __shfl_sync(0xffffffffu, v, bel ? 31 - __clz(int(bel)) : lane);
                if (t < R.ntiles)
                        carry[R.item_base + t] = bel ? nb : c;
                if (nz)
                        c = __shfl_sync(0xffffffffu, v, 31 - __clz(int(nz)));
        }
}

size_t isect_smem_bytes() {
        return size_t(kIsectWarps) * kIsectWarpBytes;
}

cudaError_t launch_isect(const IsectParams &P, bool lucene, bool passb, int num_sms, cudaStream_t stream) {
        const void *fn = lucene ? (passb ? (const void *)k_isect<true, true> : (const void *)k_isect<true, false>)
                                : (passb ? (const void *)k_isect<false, true> : (const void *)k_isect<false, false>);
        const size_t smem = isect_smem_bytes();
        cudaError_t  e    = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
        if (e != cudaSuccess)
                return e;
        int per = 0;
        if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, fn, kIsectWarps * 32, smem)) != cudaSuccess)
                return e;
        const uint32_t want = (P.total_items + kIsectWarps - 1u) / kIsectWarps;
        const uint32_t grid = std::max(1u, std::min(want, uint32_t(std::max(per, 1) * num_sms)));
        void *         args[] = {(void *)&P};
        return cudaLaunchKernel(fn, dim3(grid), dim3(kIsectWarps * 32), args, smem, stream);
}

cudaError_t launch_isect_compact(const IsectParams &P, uint64_t total_slots, const uint64_t *base, uint32_t *cursor, unsigned long long *out_mask, uint32_t *out_first,
                                 int num_sms, cudaStream_t stream) {
        if (!total_slots)
                return cudaSuccess;
        const uint64_t want = (total_slots + 255u) / 256u;
        k_isect_compact<<<unsigned(std::min<uint64_t>(want, uint64_t(num_sms) * 16u)), 256, 0, stream>>>(P, total_slots, base, cursor, out_mask, out_first);
        return cudaGetLastError();
}

cudaError_t launch_isect_carry(const IsectParams &P, unsigned long long *carry, cudaStream_t stream) {
        if (!P.nreq)
                return cudaSuccess;
        k_isect_carry<<<(P.nreq + 7u) / 8u, 256, 0, stream>>>(P, carry);
        return cudaGetLastError();
}
