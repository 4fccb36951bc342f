// Percolator kernels (trn_percolate, engine.cu; DESIGN.md §4): match a batch of documents against every registered query.
// Included by kernels.cu inside namespace trn.
//
// One CTA per document (grid-stride over the launch's documents; short and long documents run in separate launches so that the shared
// tables of the short ones stay small):
//   staging     the tokens go to shared memory; a shared open-addressing table holds the document's distinct known terms
//   candidates  the anchored lists (PercParams::csr) of the distinct terms, concatenated through a block scan over the table's slots, then the
//               unanchored queries: one flat list, one thread per entry.  A query anchored on several of the document's terms is evaluated
//               at its first anchor present: an entry with ordinal j skips when any of the query's first j anchors is on the document
//   evaluation  the query's post-order program over a 64-bit stack of presence bits; a phrase first looks its terms up in the table, then
//               tries every position of its cheapest term against the token array
//   output      k_perc<false> counts matches and evaluated pairs; the host scans the counts (launch_enc_scan); k_perc<true> evaluates again
//               and writes: up to kPercSortCap ids sorted in shared memory (bitonic), more through a zeroed bitmap over the query ids that
//               the CTA emits in order
static constexpr int kPercThreads = 256;

__device__ __forceinline__ uint32_t perc_hash(uint32_t t) {
        return t * 0x9E3779B1u;
}

__device__ __forceinline__ bool perc_present(const uint32_t *keys, uint32_t H, uint32_t t) {
        uint32_t s = perc_hash(t) & (H - 1u);
        for (;;) {
                const uint32_t k = keys[s];
                if (k == t)
                        return true;
                if (k == kEmptyTerm)
                        return false;
                s = (s + 1u) & (H - 1u);
        }
}

__device__ __forceinline__ bool perc_phrase(const PercParams &P, const PercOp &o, const uint32_t *tok, uint32_t L, const uint32_t *keys, uint32_t H) {
        const uint32_t *pt = P.phrase_terms + o.term;
        const uint32_t  n = o.n, j = o.arg;
        if (n > L)
                return false;
        for (uint32_t k = 0; k < n; ++k)
                if (!perc_present(keys, H, pt[k]))
                        return false;
        const uint32_t a = pt[j];
        for (uint32_t p = j; p + n - j <= L; ++p) {
                if (tok[p] != a)
                        continue;
                uint32_t k = 0;
                while (k < n && tok[p - j + k] == pt[k])
                        ++k;
                if (k == n)
                        return true;
        }
        return false;
}

__device__ __forceinline__ bool perc_eval(const PercParams &P, uint32_t q, const uint32_t *tok, uint32_t L, const uint32_t *keys, uint32_t H) {
        const PercQuery Q  = P.queries[q];
        uint64_t        st = 0;
        for (uint32_t i = 0; i < Q.nops; ++i) {
                const PercOp   o    = P.ops[Q.op_begin + i];
                const uint64_t mask = o.n >= 64 ? ~0ull : ((1ull << o.n) - 1ull);
                const uint64_t top  = st & mask;
                bool           v;
                switch (o.op) {
                case PERC_TERM: v = perc_present(keys, H, o.term); break;
                case PERC_PHRASE: v = perc_phrase(P, o, tok, L, keys, H); break;
                case PERC_CONST: v = o.term != 0; break;
                case PERC_AND: v = top == mask; break;
                case PERC_OR: v = top != 0; break;
                case PERC_NOT: v = ((top >> (o.n - 1u)) & 1ull) && !(top & (mask >> 1)); break;
                case PERC_OPT: v = (top >> (o.n - 1u)) & 1ull; break;
                default: v = o.arg != 0 && uint32_t(__popcll(top)) >= o.arg; break; // PERC_SOME
                }
                if (o.op >= PERC_AND)
                        st = o.n >= 64 ? 0ull : (st >> o.n);
                st = (st << 1) | uint64_t(v);
        }
        return st & 1ull;
}

// exclusive block scan of one value per thread; returns the thread's prefix, *total the sum
__device__ __forceinline__ uint32_t perc_block_scan(uint32_t v, uint32_t *warp_sums, uint32_t *total) {
        const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        uint32_t  x    = v;
        for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= o)
                        x += y;
        }
        if (lane == 31)
                warp_sums[w] = x;
        __syncthreads();
        if (w == 0) {
                uint32_t s = lane < kPercThreads / 32 ? warp_sums[lane] : 0u;
                for (int o = 1; o < 32; o <<= 1) {
                        const uint32_t y = __shfl_up_sync(0xffffffffu, s, o);
                        if (lane >= o)
                                s += y;
                }
                if (lane < kPercThreads / 32)
                        warp_sums[lane] = s;
        }
        __syncthreads();
        const uint32_t base = w ? warp_sums[w - 1] : 0u;
        *total              = warp_sums[kPercThreads / 32 - 1];
        __syncthreads();
        return base + x - v;
}

template <bool WRITE>
__global__ void __launch_bounds__(kPercThreads, 1) k_perc(const PercParams P) {
        extern __shared__ uint32_t sm[];
        uint32_t *                 tok  = sm;
        uint32_t *                 keys = tok + ((P.max_len + 3u) & ~3u);
        uint32_t *                 scan = keys + P.max_hash;      // max_hash + 1
        uint32_t *                 ids  = scan + P.max_hash + 4u; // WRITE: kPercSortCap
        __shared__ uint32_t        warp_sums[kPercThreads / 32];
        __shared__ uint32_t        s_cnt;
        __shared__ unsigned long long s_cand;
        const uint32_t             tid = threadIdx.x;

        for (uint32_t di = blockIdx.x; di < P.ndocs; di += gridDim.x) {
                const uint32_t d = P.docs[di];
                const uint64_t b = P.doc_off[d];
                const uint32_t L = uint32_t(P.doc_off[d + 1] - b);
                const uint32_t H = perc_hash_slots(L);
                if (tid == 0) {
                        s_cnt  = 0;
                        s_cand = 0;
                }
                for (uint32_t i = tid; i < L; i += kPercThreads)
                        tok[i] = P.tokens[b + i];
                for (uint32_t s = tid; s < H; s += kPercThreads)
                        keys[s] = kEmptyTerm;
                __syncthreads();
                for (uint32_t i = tid; i < L; i += kPercThreads) {
                        const uint32_t t = tok[i];
                        if (t == kEmptyTerm)
                                continue;
                        uint32_t s = perc_hash(t) & (H - 1u);
                        for (;;) {
                                const uint32_t prev = atomicCAS(&keys[s], kEmptyTerm, t);
                                if (prev == kEmptyTerm || prev == t)
                                        break;
                                s = (s + 1u) & (H - 1u);
                        }
                }
                __syncthreads();
                // the anchored entries of the table's slots, placed by an exclusive scan (each thread sums a run of consecutive slots)
                const uint32_t per = (H + kPercThreads - 1u) / kPercThreads, s0 = tid * per, s1 = min(H, s0 + per);
                uint32_t       mine{0};
                for (uint32_t s = s0; s < s1; ++s) {
                        const uint32_t t = keys[s];
                        if (t != kEmptyTerm)
                                mine += P.csr_off[t + 1] - P.csr_off[t];
                }
                uint32_t       nanch;
                uint32_t       run = perc_block_scan(mine, warp_sums, &nanch);
                for (uint32_t s = s0; s < s1; ++s) {
                        scan[s]        = run;
                        const uint32_t t = keys[s];
                        if (t != kEmptyTerm)
                                run += P.csr_off[t + 1] - P.csr_off[t];
                }
                __syncthreads();
                const uint32_t n = nanch + P.nunanchored;
                const bool     dense = WRITE && P.counts[d] > kPercSortCap;
                uint32_t *     bm    = dense ? P.bitmaps + uint64_t(P.dense_slot[d]) * P.bitmap_words : nullptr;
                uint32_t       cnt{0}, cand{0};
                for (uint32_t e = tid; e < n; e += kPercThreads) {
                        uint32_t q;
                        if (e < nanch) {
                                uint32_t lo = 0, hi = H; // the last slot whose run starts at or before e
                                while (hi - lo > 1u) {
                                        const uint32_t mid = (lo + hi) >> 1;
                                        if (scan[mid] <= e)
                                                lo = mid;
                                        else
                                                hi = mid;
                                }
                                const PercEntry E = P.csr[P.csr_off[keys[lo]] + (e - scan[lo])];
                                q                 = E.query;
                                const uint32_t *cv = P.covers + P.queries[q].cover_begin;
                                bool            earlier{false};
                                for (uint32_t j = 0; j < E.ordinal && !earlier; ++j)
                                        earlier = perc_present(keys, H, cv[j]);
                                if (earlier)
                                        continue;
                        } else
                                q = P.unanchored[e - nanch];
                        ++cand;
                        if (!perc_eval(P, q, tok, L, keys, H))
                                continue;
                        if (!WRITE)
                                ++cnt;
                        else if (dense)
                                atomicOr(&bm[q >> 5], 1u << (q & 31u));
                        else
                                ids[atomicAdd(&s_cnt, 1u)] = q;
                }
                if (!WRITE) {
                        atomicAdd(&s_cnt, cnt);
                        atomicAdd(&s_cand, (unsigned long long)cand);
                        __syncthreads();
                        if (tid == 0) {
                                P.counts[d] = s_cnt;
                                atomicAdd(P.candidates, s_cand);
                        }
                } else if (!dense) {
                        // bitonic sort of the ids in shared memory, padded to a power of two with kEmptyTerm
                        __syncthreads();
                        const uint32_t c = s_cnt;
                        uint32_t       m = 1;
                        while (m < c)
                                m <<= 1;
                        for (uint32_t i = c + tid; i < m; i += kPercThreads)
                                ids[i] = kEmptyTerm;
                        __syncthreads();
                        for (uint32_t k = 2; k <= m; k <<= 1)
                                for (uint32_t j = k >> 1; j > 0; j >>= 1) {
                                        for (uint32_t i = tid; i < m; i += kPercThreads) {
                                                const uint32_t x = i ^ j;
                                                if (x > i) {
                                                        const uint32_t a = ids[i], bb = ids[x];
                                                        if (((i & k) == 0) == (a > bb)) {
                                                                ids[i] = bb;
                                                                ids[x] = a;
                                                        }
                                                }
                                        }
                                        __syncthreads();
                                }
                        uint32_t *out = P.out + P.out_off[d];
                        for (uint32_t i = tid; i < c; i += kPercThreads)
                                out[i] = ids[i];
                } else {
                        // the bitmap in query-id order: each thread emits a run of consecutive words
                        __syncthreads();
                        const uint32_t W = P.bitmap_words, wper = (W + kPercThreads - 1u) / kPercThreads, w0 = min(W, tid * wper), w1 = min(W, w0 + wper);
                        uint32_t       pc{0};
                        for (uint32_t w = w0; w < w1; ++w)
                                pc += __popc(__ldcg(&bm[w]));
                        uint32_t  tot;
                        uint32_t  at  = perc_block_scan(pc, warp_sums, &tot);
                        uint32_t *out = P.out + P.out_off[d];
                        for (uint32_t w = w0; w < w1; ++w)
                                for (uint32_t x = __ldcg(&bm[w]); x; x &= x - 1u)
                                        out[at++] = (w << 5) + uint32_t(__ffs(int(x)) - 1);
                }
                __syncthreads(); // the shared tables are rebuilt for the next document
        }
}

size_t perc_smem_bytes(uint32_t max_len, uint32_t max_hash, bool write) {
        return (size_t((max_len + 3u) & ~3u) + 2u * max_hash + 4u + (write ? kPercSortCap : 0u)) * 4u;
}

cudaError_t launch_perc(const PercParams &P, bool write, int num_sms, cudaStream_t stream) {
        if (!P.ndocs)
                return cudaSuccess;
        const void * fn   = write ? (const void *)k_perc<true> : (const void *)k_perc<false>;
        const size_t smem = perc_smem_bytes(P.max_len, P.max_hash, write);
        cudaError_t  e    = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
        if (e != cudaSuccess)
                return e;
        int per = 0;
        if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, fn, kPercThreads, smem)) != cudaSuccess)
                return e;
        const uint32_t grid   = std::max(1u, std::min(P.ndocs, uint32_t(std::max(per, 1) * num_sms)));
        void *         args[] = {(void *)&P};
        return cudaLaunchKernel(fn, dim3(grid), dim3(kPercThreads), args, smem, stream);
}
