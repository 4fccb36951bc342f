// trn_merge_sources / trn_merge_sources_payloads on the device (included by kernels.cu): the postings of every merged term are decoded from
// the sources' own bytes, the postings the reference's merge() writes are kept and ranked without a sort, and the survivors are scattered
// into the term-major layout the device encoders read.  One thread per block (decode), per posting (hits, keep, rank) or per output posting
// (hits scatter); every list is read through the load-time block / hits directories of its source (MergeParams::views), so a thread starts
// anywhere.
//
// Keep and rank (the newest holder of a docID decides, merge.cpp:333-365 / google_codec.cpp IndexSession::merge): posting (p, d) of a
// re-encoded term is kept iff no newer participant of the term holds d (binary search in its decoded docIDs) and d is not in p's
// registry (binary search in the sorted updated docIDs; masked iff the newest candidate listing d is newer than p).  With kscan the
// exclusive scan of the keep flags, its output rank is its kept rank in its own list + the kept postings below d of every other
// participant: the kept docIDs of one term are distinct, so the ranks are a permutation — a k-way merge without a sort.
//
// Payloads (materialize_hits + new_hit(pos, {payload, len}), merge.cpp:221-232, 352-361): the positions pass records whether a kept hit
// carries one.  Only then, and only when the call takes payloads, a per-hit length and payload array is allocated beside the positions and
// the PAYLOADS form of the same pass fills all three; k_merge_hits<true> carries them to the output order and the encoders' payload
// instantiations write them.  A merge without payload hits runs the payload-free forms and allocates nothing more.

__device__ __forceinline__ uint32_t mg_list_of(const unsigned long long *begin, uint32_t n, unsigned long long i) { // last l with begin[l] <= i
        uint32_t lo = 0, hi = n;
        while (hi - lo > 1) {
                const uint32_t m = (lo + hi) >> 1;
                if (begin[m] <= i)
                        lo = m;
                else
                        hi = m;
        }
        return lo;
}
__device__ __forceinline__ uint64_t mg_lower_bound(const uint32_t *a, uint64_t n, uint32_t d) {
        uint64_t lo = 0, hi = n;
        while (lo < hi) {
                const uint64_t m = (lo + hi) >> 1;
                if (a[m] < d)
                        lo = m + 1;
                else
                        hi = m;
        }
        return lo;
}
__device__ __forceinline__ PhraseTerm mg_term(const MergeList &L) {
        PhraseTerm t;
        t.dir    = L.t.dir_begin;
        t.nb     = L.t.nblocks;
        t.docs   = L.t.documents;
        t.first  = L.t.first_doc;
        t.last   = L.t.last_doc;
        t.tfb    = L.t.tf_begin;
        t.tfbase = L.t.tf_base;
        t.tfs    = L.t.tf_shift;
        t.id     = L.term;
        return t;
}

// one thread per block of a list: its docIDs and freqs (GOOGLE google_codec.cpp:596-639: n - 1 doc deltas, the last docID from the
// directory, n freqs; LUCENE lucene_codec.cpp:515-558: a full block is a deltas and a freqs int-block, the tail varbyte pairs)
__global__ void __launch_bounds__(kThreads) k_merge_decode_blocks(MergeParams P) {
        const unsigned long long g = blockIdx.x * (unsigned long long)kThreads + threadIdx.x;
        if (g >= P.nblocks)
                return;
        const uint32_t   l = mg_list_of(P.list_blk, P.nlists, g);
        const MergeList &L = P.lists[l];
        const HitsView  &V = P.views[L.view];
        const uint32_t   b = uint32_t(g - P.list_blk[l]);
        const uint32_t   dir = L.t.dir_begin;
        const uint32_t   prev = b ? V.blk_last[dir + b - 1u] : 0u;
        const uint8_t   *p    = V.index + V.blk_off[dir + b];
        const bool       hits = L.reencode;
        if (V.codec == 0) {
                const uint32_t n   = (b + 1u == L.t.nblocks) ? (L.t.documents - 32u * (L.t.nblocks - 1u)) : 32u;
                const uint64_t o   = P.list_post[l] + 32ull * b;
                uint32_t       doc = prev;
                for (uint32_t i = 0; i + 1u < n; ++i) {
                        doc += varbyte_get(p);
                        P.docids[o + i] = doc;
                }
                P.docids[o + n - 1u] = V.blk_last[dir + b];
                for (uint32_t i = 0; i < n; ++i) {
                        const uint32_t f = varbyte_get(p) & 0xffffu; // uint16_t in the reference (codecs.h:217)
                        P.freqs[o + i]   = f;
                        P.hcount[o + i]  = hits ? f : 0u;
                }
                return;
        }
        const uint64_t o = P.list_post[l] + 128ull * b;
        if (b < (L.t.documents >> 7)) {
                PforRef D;
                D.init(p);
                uint32_t doc = prev, e = 0;
                for (uint32_t i = 0; i < 128u; ++i) {
                        doc += D.get(i, e);
                        P.docids[o + i] = doc;
                }
                PforRef F;
                F.init(D.end());
                e = 0;
                for (uint32_t i = 0; i < 128u; ++i) {
                        const uint32_t f = F.get(i, e) & 0xffffu;
                        P.freqs[o + i]   = f;
                        P.hcount[o + i]  = hits ? f : 0u;
                }
                return;
        }
        const uint32_t n   = L.t.documents & 127u;
        uint32_t       doc = prev;
        for (uint32_t i = 0; i < n; ++i) {
                doc += varbyte_get(p);
                const uint32_t f = varbyte_get(p) & 0xffffu;
                P.docids[o + i]  = doc;
                P.freqs[o + i]   = f;
                P.hcount[o + i]  = hits ? f : 0u;
        }
}

// one thread per KEPT posting of a re-encoded list (k_merge_keep zeroes hcount of the others): its positions (hitcursor.h HitWalker, the
// reader the exec paths use) at hoff[i].  Recorded, as the first such posting: error[0] a hit with a payload (whether the PAYLOADS pass
// runs; trn_merge_sources refuses it), error[1] a hit at position 0 without a payload or above 16383 (the encoders take neither),
// error[2] a stored payload length above 8 (a malformed source: the reference's payload is a u64).  PAYLOADS also writes each hit's
// length to plens and its payload to pays, masked to the low `len` bytes: a GOOGLE walker keeps the high bytes of an earlier, longer
// payload of the same document (materialize_hits), and the arrays hold what a reader hands back.  Postings that are not written are never
// looked at, as merge() never materialises their hits; a LUCENE walker that starts inside a 128-hit block skips the payload bytes of the
// block's earlier hits by their lengths (HitWalker::lucene_block), so the bytes of a masked or older posting there are never read either.
template <bool PAYLOADS>
__global__ void __launch_bounds__(kThreads) k_merge_decode_hits(MergeParams P) {
        const unsigned long long i = blockIdx.x * (unsigned long long)kThreads + threadIdx.x;
        if (i >= P.nposts || !P.hcount[i])
                return;
        const MergeList &L = P.lists[mg_list_of(P.list_post, P.nlists, i)];
        HitWalker        w;
        w.init(P.views[L.view], mg_term(L), P.docids[i]);
        const uint32_t   f = P.hcount[i];
        uint32_t        *o = P.positions + P.hoff[i];
        uint32_t any = 0, bad = 0, big = 0; // flags tested after the loop: an atomic inside it costs a spill
        for (uint32_t h = 0; h < f; ++h) {
                uint32_t len;
                const uint32_t pos = w.next(len);
                o[h] = pos;
                if constexpr (PAYLOADS) {
                        P.plens[P.hoff[i] + h] = uint8_t(len);
                        P.pays[P.hoff[i] + h]  = len >= 8u ? w.payload : w.payload & ((1ull << (8u * len)) - 1ull);
                }
                any |= len;
                bad |= (pos == 0u && !len) || pos > 16383u;
                big |= len > 8u;
        }
        if (any)
                atomicMin(P.error, i);
        if (bad)
                atomicMin(P.error + 1, i);
        if (big)
                atomicMin(P.error + 2, i);
}

// one thread per posting (before the hits are decoded): keep flag (re-encoded lists) and the docs_cnt bitmap (every output posting, appended ones included)
__global__ void __launch_bounds__(kThreads) k_merge_keep(MergeParams P) {
        const unsigned long long i = blockIdx.x * (unsigned long long)kThreads + threadIdx.x;
        if (i >= P.nposts)
                return;
        const uint32_t   l = mg_list_of(P.list_post, P.nlists, i);
        const MergeList &L = P.lists[l];
        const uint32_t   d = P.docids[i];
        uint32_t         keep = 1;
        if (L.reencode) {
                const uint64_t u = mg_lower_bound(P.upd_docid, P.nupd, d);
                if (u < P.nupd && P.upd_docid[u] == d && P.upd_first[u] < L.cand)
                        keep = 0;
                for (uint32_t q = l - L.rank; keep && q < l; ++q) { // the newer participants of the same term
                        const uint64_t b = P.list_post[q], n = P.list_post[q + 1] - b;
                        const uint64_t k = mg_lower_bound(P.docids + b, n, d);
                        keep = !(k < n && P.docids[b + k] == d);
                }
        }
        P.keep[i] = L.reencode ? keep : 0u;
        if (!keep)
                P.hcount[i] = 0;
        if (keep)
                atomicOr(P.bitmap + (d >> 5), 1u << (d & 31u));
}

// one thread per kept posting: its output place = the term's first output posting + its rank; docID, freq and source posting there
__global__ void __launch_bounds__(kThreads) k_merge_scatter(MergeParams P) {
        const unsigned long long i = blockIdx.x * (unsigned long long)kThreads + threadIdx.x;
        if (i >= P.nposts || !P.keep[i])
                return;
        const uint32_t   l = mg_list_of(P.list_post, P.nlists, i);
        const MergeList &L = P.lists[l];
        const uint32_t   d = P.docids[i];
        const uint32_t   first = l - L.rank;
        unsigned long long r = P.kscan[P.list_post[first]] + (P.kscan[i] - P.kscan[P.list_post[l]]);
        for (uint32_t q = first; q < first + L.nparts; ++q)
                if (q != l) {
                        const uint64_t b = P.list_post[q];
                        r += P.kscan[b + mg_lower_bound(P.docids + b, P.list_post[q + 1] - b, d)] - P.kscan[b];
                }
        P.out_docids[r] = d;
        P.out_freqs[r]  = P.freqs[i];
        P.out_src[r]    = i;
}

// one thread per output posting: its positions (PAYLOADS: and their lengths and payloads) from the decoded hits (out_hoff = the scan of
// the output freqs)
template <bool PAYLOADS>
__global__ void __launch_bounds__(kThreads) k_merge_hits(MergeParams P, unsigned long long nout) {
        const unsigned long long j = blockIdx.x * (unsigned long long)kThreads + threadIdx.x;
        if (j >= nout)
                return;
        const unsigned long long i = P.out_src[j];
        const uint32_t           f = P.out_freqs[j];
        const uint32_t          *s = P.positions + P.hoff[i];
        uint32_t                *o = P.out_positions + P.out_hoff[j];
        for (uint32_t h = 0; h < f; ++h)
                o[h] = s[h];
        if constexpr (PAYLOADS)
                for (uint32_t h = 0; h < f; ++h) {
                        P.out_plens[P.out_hoff[j] + h] = P.plens[P.hoff[i] + h];
                        P.out_pays[P.out_hoff[j] + h]  = P.pays[P.hoff[i] + h];
                }
}

__global__ void __launch_bounds__(kThreads) k_merge_gather(const unsigned long long *a, const unsigned long long *idx, uint32_t n, unsigned long long *out) {
        const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
        if (i < n)
                out[i] = a[idx[i]];
}

__global__ void __launch_bounds__(kThreads) k_merge_popcount(const uint32_t *bitmap, unsigned long long nwords, unsigned long long *count) {
        unsigned long long c = 0;
        for (unsigned long long w = blockIdx.x * (unsigned long long)kThreads + threadIdx.x; w < nwords; w += (unsigned long long)gridDim.x * kThreads)
                c += __popc(bitmap[w]);
        for (int o = 16; o; o >>= 1)
                c += __shfl_down_sync(0xffffffffu, c, o);
        if ((threadIdx.x & 31u) == 0 && c)
                atomicAdd(count, c);
}

// the assembly: one CTA per copy segment (an index chunk or a positions chunk) into the output; a LUCENE index chunk gets its final
// hitsDataOffset in its first four bytes (lucene_codec.cpp:139-161)
__global__ void __launch_bounds__(kThreads) k_merge_assemble(const MergeCopy *segs, uint8_t *index_out, uint8_t *hits_out) {
        const MergeCopy S   = segs[blockIdx.x];
        uint8_t        *dst = (S.to_hits ? hits_out : index_out) + S.dst;
        for (unsigned long long k = threadIdx.x; k < S.len; k += kThreads)
                dst[k] = (S.header && k < 4) ? uint8_t(S.hits_off >> (8u * k)) : S.src[k];
}

cudaError_t launch_merge_decode(const MergeParams &P, cudaStream_t stream) {
        if (P.nblocks)
                k_merge_decode_blocks<<<unsigned((P.nblocks + kThreads - 1) / kThreads), kThreads, 0, stream>>>(P);
        return cudaGetLastError();
}
cudaError_t launch_merge_hits_decode(const MergeParams &P, bool payloads, cudaStream_t stream) {
        if (P.nposts && payloads)
                k_merge_decode_hits<true><<<unsigned((P.nposts + kThreads - 1) / kThreads), kThreads, 0, stream>>>(P);
        else if (P.nposts)
                k_merge_decode_hits<false><<<unsigned((P.nposts + kThreads - 1) / kThreads), kThreads, 0, stream>>>(P);
        return cudaGetLastError();
}
cudaError_t launch_merge_keep(const MergeParams &P, cudaStream_t stream) {
        if (P.nposts)
                k_merge_keep<<<unsigned((P.nposts + kThreads - 1) / kThreads), kThreads, 0, stream>>>(P);
        return cudaGetLastError();
}
cudaError_t launch_merge_scatter(const MergeParams &P, cudaStream_t stream) {
        if (P.nposts)
                k_merge_scatter<<<unsigned((P.nposts + kThreads - 1) / kThreads), kThreads, 0, stream>>>(P);
        return cudaGetLastError();
}
cudaError_t launch_merge_out_hits(const MergeParams &P, uint64_t nout, bool payloads, cudaStream_t stream) {
        if (nout && payloads)
                k_merge_hits<true><<<unsigned((nout + kThreads - 1) / kThreads), kThreads, 0, stream>>>(P, nout);
        else if (nout)
                k_merge_hits<false><<<unsigned((nout + kThreads - 1) / kThreads), kThreads, 0, stream>>>(P, nout);
        return cudaGetLastError();
}
cudaError_t launch_merge_gather(const unsigned long long *a, const unsigned long long *idx, uint32_t n, unsigned long long *out, cudaStream_t stream) {
        if (n)
                k_merge_gather<<<(n + kThreads - 1) / kThreads, kThreads, 0, stream>>>(a, idx, n, out);
        return cudaGetLastError();
}
cudaError_t launch_merge_popcount(const uint32_t *bitmap, uint64_t nwords, unsigned long long *count, cudaStream_t stream) {
        k_merge_popcount<<<unsigned(std::min<uint64_t>(1024, (nwords + kThreads - 1) / kThreads + 1)), kThreads, 0, stream>>>(bitmap, nwords, count);
        return cudaGetLastError();
}
cudaError_t launch_merge_assemble(const MergeCopy *segs, uint32_t nsegs, uint8_t *index_out, uint8_t *hits_out, cudaStream_t stream) {
        if (nsegs)
                k_merge_assemble<<<nsegs, kThreads, 0, stream>>>(segs, index_out, hits_out);
        return cudaGetLastError();
}
