// Indexer kernels (trn_index_documents, engine.cu; DESIGN.md §4): a batch of tokenised documents -> term-major postings in the layout the
// device encoders read.  (Included by kernels.cu.)
//
// Replaces (reference): SegmentIndexSession's per-document hit sort (indexer.cpp:54-57) and commit()'s collect / bucket / sort of the
// (term, document) records (indexer.cpp:337-420).  The inversion is one keys-only sort:
//   key         term_order << 40 | doc_rank << 14 | position.  term_order = the term's place in commit()'s encode order (buckets by transient
//               id & 31, ascending id inside a bucket, indexer.cpp:388,402-410,423); doc_rank = the document's rank in docID order; position
//               < 2^14 (Limits::MaxPosition).  Sorted keys ARE the index order: terms, inside a term ascending docIDs, inside a posting
//               ascending positions.
//   documents   the docIDs are sorted with the same radix sort (key docID << 32 | ordinal); neighbours show duplicates and docID 0.
//   token->doc  every token finds its document by a binary search over doc_offsets (at most 27 probes of an array that stays in L2): the work
//               per token does not depend on how long the documents are, which one warp per document cannot say of a batch that mixes
//               one-token and 16 383-token documents.
//   radix sort  LSD, one pass per group of up to 8 key bits that can be non-zero (the host plans the passes, IndexPass): k_radix_hist counts
//               the digits of every 4096-key tile (digit-major counts, so one exclusive scan places every (digit, tile)), k_radix_scatter ranks
//               the tile's keys stably (per-warp __match_any_sync ranks over per-warp digit counters), stages the tile in digit order in
//               shared memory and copies it out, so neighbouring threads write neighbouring keys of one digit run.
//   postings    k_post_flags marks the tokens that open a posting / a term; two scans number them; k_post_write emits docids, the first hit
//               of every posting, positions, term_begin and the terms' orders; k_post_freqs derives the freqs and checks the u16 limits.
//   payloads    the key has no spare bit, so a call with payloads sorts a u32 token ordinal beside every key (the VALUES instantiation of
//               k_radix_scatter; the keys-only passes are the ones a call without payloads runs) and k_post_write gathers every hit's
//               payload size and bytes through it.  Equal keys with different payloads are refused: the reference orders them with an
//               unstable sort (indexer.cpp:55-57).
#pragma once

static constexpr uint32_t kRadixTile    = 4096; // keys per CTA of the sort kernels (256 threads x 16)
static constexpr uint32_t kRadixThreads = 256;
static constexpr uint32_t kRadixPer     = kRadixTile / kRadixThreads;

__global__ void __launch_bounds__(256) k_index_doc_keys(const uint32_t *docids, uint32_t ndocs, unsigned long long *keys) {
        const uint32_t i = blockIdx.x * 256u + threadIdx.x;
        if (i < ndocs)
                keys[i] = (uint64_t(docids[i]) << 32) | i;
}

// sorted (docID, ordinal) -> rank of every document, docIDs by rank; errors[IDX_ERR_DOC0 / IDX_ERR_DUP] = the lowest offending ordinal
__global__ void __launch_bounds__(256) k_index_doc_ranks(const unsigned long long *keys, uint32_t ndocs, uint32_t *rank_of, uint32_t *docid_of,
                                                          unsigned long long *errors) {
        const uint32_t i = blockIdx.x * 256u + threadIdx.x;
        if (i >= ndocs)
                return;
        const uint64_t k   = keys[i];
        const uint32_t doc = uint32_t(k >> 32), ord = uint32_t(k);
        if (doc == 0)
                atomicMin(errors + IDX_ERR_DOC0, (unsigned long long)ord);
        if (i && uint32_t(keys[i - 1] >> 32) == doc)
                atomicMin(errors + IDX_ERR_DUP, (unsigned long long)ord);
        rank_of[ord] = i;
        docid_of[i]  = doc;
}

// one thread per token: its document (binary search), its key; errors[] = the lowest offending token of every kind
__global__ void __launch_bounds__(256) k_index_keys(IndexParams P) {
        const uint64_t i = uint64_t(blockIdx.x) * 256u + threadIdx.x;
        if (i >= P.ntokens)
                return;
        // the last document whose first token is <= i (empty documents share their successor's offset and are passed over)
        uint32_t lo = 0, hi = P.ndocs;
        while (hi - lo > 1) {
                const uint32_t mid = lo + (hi - lo) / 2;
                if (P.doc_off[mid] <= i)
                        lo = mid;
                else
                        hi = mid;
        }
        const uint32_t t   = P.tokens[i];
        const uint32_t pos = P.positions ? P.positions[i] : uint32_t(i - P.doc_off[lo]) + 1u;
        if (t >= P.nterms) {
                atomicMin(P.errors + IDX_ERR_TOKEN, (unsigned long long)i);
                P.keys[i] = 0;
                return;
        }
        const uint32_t len = P.plens ? P.plens[i] : 0u;
        if (P.plens) {
                P.ords[i] = uint32_t(i);
                if (len > 8u)
                        atomicMin(P.errors + IDX_ERR_PAYLEN, (unsigned long long)i);
        }
        if (pos == 0 && len == 0) // a position-0 hit with a payload is written and counted (google_codec.cpp:42-45)
                atomicMin(P.errors + IDX_ERR_POS0, (unsigned long long)i);
        else if (pos >= 16384u)
                atomicMin(P.errors + IDX_ERR_POS, (unsigned long long)i);
        P.keys[i] = (uint64_t(index_term_order(t, P.nterms)) << 40) | (uint64_t(P.rank_of[lo]) << 14) | (pos & 16383u);
}

// ---- radix sort pass: digit = (key >> shift) & mask
__global__ void __launch_bounds__(kRadixThreads) k_radix_hist(const unsigned long long *keys, uint64_t n, uint32_t shift, uint32_t mask, uint32_t ntiles,
                                                             uint32_t *counts /* [digit][tile] */) {
        __shared__ uint32_t s_h[256];
        s_h[threadIdx.x] = 0;
        __syncthreads();
        const uint64_t base = uint64_t(blockIdx.x) * kRadixTile;
#pragma unroll
        for (uint32_t k = 0; k < kRadixPer; ++k) {
                const uint64_t i = base + k * kRadixThreads + threadIdx.x;
                if (i < n)
                        atomicAdd(&s_h[uint32_t(keys[i] >> shift) & mask], 1u);
        }
        __syncthreads();
        if (threadIdx.x <= mask)
                counts[size_t(threadIdx.x) * ntiles + blockIdx.x] = s_h[threadIdx.x];
}

// VALUES: vin[] moves with the keys into vout[] (the keys' staging area holds the values once the keys are out)
template <bool VALUES = false>
__global__ void __launch_bounds__(kRadixThreads) k_radix_scatter(const unsigned long long *in, unsigned long long *out, uint64_t n, uint32_t shift, uint32_t mask,
                                                                uint32_t ntiles, const unsigned long long *offsets /* scan of counts */, const uint32_t *vin,
                                                                uint32_t *vout) {
        constexpr uint32_t W = kRadixThreads / 32, ROUNDS = kRadixTile / kRadixThreads; // a warp owns ROUNDS x 32 consecutive keys of the tile
        __shared__ unsigned long long s_stage[kRadixTile];
        __shared__ unsigned long long s_gofs[256];
        __shared__ uint32_t           s_wcnt[W][256]; // keys of every digit in every warp's part, then the part's first place in the digit's run
        __shared__ uint32_t           s_start[256];   // first staged place of every digit
        const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const uint64_t base = uint64_t(blockIdx.x) * kRadixTile;
        const uint32_t cnt  = uint32_t(min(uint64_t(kRadixTile), n - base));
        for (uint32_t w = 0; w < W; ++w)
                s_wcnt[w][threadIdx.x] = 0;
        s_gofs[threadIdx.x] = threadIdx.x <= mask ? offsets[size_t(threadIdx.x) * ntiles + blockIdx.x] : 0ull;
        __syncthreads();
        unsigned long long key[ROUNDS];
        uint16_t           rnk[ROUNDS];
#pragma unroll
        for (uint32_t r = 0; r < ROUNDS; ++r) {
                const uint32_t j     = warp * (ROUNDS * 32u) + r * 32u + lane;
                const bool     valid = j < cnt;
                key[r]               = valid ? in[base + j] : 0ull;
                const uint32_t d     = valid ? (uint32_t(key[r] >> shift) & mask) : 256u; // keys past the end form their own group and count nowhere
                const uint32_t peers = __match_any_sync(0xffffffffu, d);
                const uint32_t before = __popc(peers & ((1u << lane) - 1u));
                uint32_t       at{0};
                if (valid)
                        at = s_wcnt[warp][d];
                __syncwarp();
                if (valid && before == 0)
                        s_wcnt[warp][d] = at + __popc(peers);
                __syncwarp();
                rnk[r] = uint16_t(at + before);
        }
        __syncthreads();
        // digit `threadIdx.x`: its keys in the tile, the first place of every warp's part inside its run
        uint32_t total{0};
        for (uint32_t w = 0; w < W; ++w) {
                const uint32_t v       = s_wcnt[w][threadIdx.x];
                s_wcnt[w][threadIdx.x] = total;
                total += v;
        }
        // exclusive scan of the digit totals over the CTA
        uint32_t incl = total;
        for (int s = 1; s < 32; s <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, incl, s);
                if (lane >= uint32_t(s))
                        incl += y;
        }
        __shared__ uint32_t s_wsum[W];
        if (lane == 31)
                s_wsum[warp] = incl;
        __syncthreads();
        uint32_t wbase{0};
        for (uint32_t w = 0; w < warp; ++w)
                wbase += s_wsum[w];
        s_start[threadIdx.x] = wbase + incl - total;
        __syncthreads();
#pragma unroll
        for (uint32_t r = 0; r < ROUNDS; ++r) {
                const uint32_t j = warp * (ROUNDS * 32u) + r * 32u + lane;
                if (j < cnt) {
                        const uint32_t d                                   = uint32_t(key[r] >> shift) & mask;
                        s_stage[s_start[d] + s_wcnt[warp][d] + rnk[r]] = key[r];
                }
        }
        __syncthreads();
        if constexpr (!VALUES) {
                for (uint32_t s = threadIdx.x; s < cnt; s += kRadixThreads) {
                        const unsigned long long k = s_stage[s];
                        const uint32_t           d = uint32_t(k >> shift) & mask;
                        out[s_gofs[d] + (s - s_start[d])] = k;
                }
        } else {
                uint64_t dst[ROUNDS]; // the place of staged entry threadIdx.x + r * kRadixThreads in out[]
#pragma unroll
                for (uint32_t r = 0; r < ROUNDS; ++r) {
                        const uint32_t s = threadIdx.x + r * kRadixThreads;
                        if (s < cnt) {
                                const unsigned long long k = s_stage[s];
                                const uint32_t           d = uint32_t(k >> shift) & mask;
                                dst[r]                     = s_gofs[d] + (s - s_start[d]);
                                out[dst[r]]                = k;
                        }
                }
                __syncthreads();
                uint32_t *s_val = reinterpret_cast<uint32_t *>(s_stage);
#pragma unroll
                for (uint32_t r = 0; r < ROUNDS; ++r) {
                        const uint32_t j = warp * (ROUNDS * 32u) + r * 32u + lane;
                        if (j < cnt) {
                                const uint32_t d                             = uint32_t(key[r] >> shift) & mask;
                                s_val[s_start[d] + s_wcnt[warp][d] + rnk[r]] = vin[base + j];
                        }
                }
                __syncthreads();
#pragma unroll
                for (uint32_t r = 0; r < ROUNDS; ++r) {
                        const uint32_t s = threadIdx.x + r * kRadixThreads;
                        if (s < cnt)
                                vout[dst[r]] = s_val[s];
                }
        }
}

// ---- postings over the sorted keys
__global__ void __launch_bounds__(256) k_post_flags(const unsigned long long *keys, uint64_t n, uint32_t *post_flag, uint32_t *term_flag) {
        const uint64_t i = uint64_t(blockIdx.x) * 256u + threadIdx.x;
        if (i >= n)
                return;
        const uint64_t k = keys[i], p = i ? keys[i - 1] : 0ull;
        post_flag[i]     = !i || (k >> 14) != (p >> 14);
        term_flag[i]     = !i || (k >> 40) != (p >> 40);
}

// with payloads (P.out_plens): ords = the sorted token ordinals; errors[IDX_ERR_PAYDUP] = the lowest sorted token whose key equals its
// predecessor's while its payload differs
__global__ void __launch_bounds__(256) k_post_write(IndexParams P, const unsigned long long *keys, const uint32_t *ords) {
        const uint64_t i = uint64_t(blockIdx.x) * 256u + threadIdx.x;
        if (i > P.ntokens)
                return;
        if (i == P.ntokens) { // the sentinels
                P.post_begin[P.post_scan[i]] = i;
                P.term_begin[P.term_scan[i]] = P.post_scan[i];
                return;
        }
        const uint64_t k = keys[i];
        P.out_positions[i] = uint32_t(k) & 16383u;
        if (P.out_plens) {
                const auto     payload_of = [&](uint32_t o, uint32_t &len) {
                        len = P.plens[o];
                        return len >= 8u ? P.payloads[o] : P.payloads[o] & ((1ull << (8u * len)) - 1ull);
                };
                uint32_t                 len;
                const unsigned long long v = payload_of(ords[i], len);
                P.out_plens[i]             = uint8_t(len);
                P.out_payloads[i]          = v;
                if (i && keys[i - 1] == k) {
                        uint32_t plen;
                        if (payload_of(ords[i - 1], plen) != v || plen != len)
                                atomicMin(P.errors + IDX_ERR_PAYDUP, (unsigned long long)i);
                }
        }
        if (P.post_flag[i]) {
                const uint64_t p    = P.post_scan[i];
                const uint32_t rank = uint32_t(k >> 14) & 0x3ffffffu;
                P.out_docids[p]     = P.docid_of[rank];
                P.post_begin[p]     = i;
                if (P.doc_terms)
                        atomicAdd(P.doc_terms + rank, 1u);
                if (P.term_flag[i]) {
                        const uint64_t j = P.term_scan[i];
                        P.term_begin[j]  = p;
                        P.term_order[j]  = uint32_t(k >> 40);
                }
        }
}

// freqs from the postings' first hits; errors[IDX_ERR_FREQ] = the lowest posting of more than 65535 hits (a uint16_t field, indexer.cpp:102-103)
__global__ void __launch_bounds__(256) k_post_freqs(IndexParams P, uint64_t nposts) {
        const uint64_t p = uint64_t(blockIdx.x) * 256u + threadIdx.x;
        if (p >= nposts)
                return;
        const uint64_t f = P.post_begin[p + 1] - P.post_begin[p];
        if (f > 65535u)
                atomicMin(P.errors + IDX_ERR_FREQ, (unsigned long long)p);
        P.out_freqs[p] = uint32_t(f);
}

// errors[IDX_ERR_DOCTERMS] = the lowest rank of a document of more than 65535 distinct terms (a uint16_t field, indexer.cpp:49,111)
__global__ void __launch_bounds__(256) k_index_doc_terms(const uint32_t *doc_terms, uint32_t ndocs, unsigned long long *errors) {
        const uint32_t i = blockIdx.x * 256u + threadIdx.x;
        if (i < ndocs && doc_terms[i] > 65535u)
                atomicMin(errors + IDX_ERR_DOCTERMS, (unsigned long long)i);
}

cudaError_t launch_index_doc_keys(const uint32_t *docids, uint32_t ndocs, unsigned long long *keys, cudaStream_t stream) {
        k_index_doc_keys<<<(ndocs + 255u) / 256u, 256, 0, stream>>>(docids, ndocs, keys);
        return cudaGetLastError();
}
cudaError_t launch_index_doc_ranks(const unsigned long long *keys, uint32_t ndocs, uint32_t *rank_of, uint32_t *docid_of, unsigned long long *errors,
                                   cudaStream_t stream) {
        k_index_doc_ranks<<<(ndocs + 255u) / 256u, 256, 0, stream>>>(keys, ndocs, rank_of, docid_of, errors);
        return cudaGetLastError();
}
cudaError_t launch_index_keys(const IndexParams &P, cudaStream_t stream) {
        if (!P.ntokens)
                return cudaSuccess;
        k_index_keys<<<unsigned((P.ntokens + 255u) / 256u), 256, 0, stream>>>(P);
        return cudaGetLastError();
}
// one pass of the sort: in -> out by the digit (key >> shift) & (2^bits - 1); counts: 2^bits x tiles u32, offsets: one more u64 than that.
// vin / vout (both or neither): a u32 per key that moves with it
cudaError_t launch_radix_pass(const unsigned long long *in, unsigned long long *out, uint64_t n, uint32_t shift, uint32_t bits, uint32_t *counts,
                              unsigned long long *partials, unsigned long long *offsets, cudaStream_t stream, const uint32_t *vin, uint32_t *vout) {
        if (!n)
                return cudaSuccess;
        const uint32_t ntiles = uint32_t((n + kRadixTile - 1) / kRadixTile), mask = (1u << bits) - 1u;
        k_radix_hist<<<ntiles, kRadixThreads, 0, stream>>>(in, n, shift, mask, ntiles, counts);
        cudaError_t e = launch_enc_scan(counts, uint64_t(mask + 1u) * ntiles, partials, offsets, stream);
        if (e != cudaSuccess)
                return e;
        if (vin)
                k_radix_scatter<true><<<ntiles, kRadixThreads, 0, stream>>>(in, out, n, shift, mask, ntiles, offsets, vin, vout);
        else
                k_radix_scatter<<<ntiles, kRadixThreads, 0, stream>>>(in, out, n, shift, mask, ntiles, offsets, nullptr, nullptr);
        return cudaGetLastError();
}
cudaError_t launch_post_flags(const unsigned long long *keys, uint64_t n, uint32_t *post_flag, uint32_t *term_flag, cudaStream_t stream) {
        if (!n)
                return cudaSuccess;
        k_post_flags<<<unsigned((n + 255u) / 256u), 256, 0, stream>>>(keys, n, post_flag, term_flag);
        return cudaGetLastError();
}
cudaError_t launch_post_write(const IndexParams &P, const unsigned long long *keys, const uint32_t *ords, cudaStream_t stream) {
        k_post_write<<<unsigned((P.ntokens + 256u) / 256u), 256, 0, stream>>>(P, keys, ords);
        return cudaGetLastError();
}
cudaError_t launch_post_freqs(const IndexParams &P, uint64_t nposts, cudaStream_t stream) {
        if (nposts)
                k_post_freqs<<<unsigned((nposts + 255u) / 256u), 256, 0, stream>>>(P, nposts);
        if (P.doc_terms)
                k_index_doc_terms<<<(P.ndocs + 255u) / 256u, 256, 0, stream>>>(P.doc_terms, P.ndocs, P.errors);
        return cudaGetLastError();
}
