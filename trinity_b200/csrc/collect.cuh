// The collect pass of the default exec mode (TRN_MODE_MATCHED_TERMS; Included by kernels.cu, after phrase.cuh).
//
// The docs pass (k_exec_docs, the DocumentsOnly routes with the root-filter quirk off) leaves every query's matches, ascending, in HBM.
// Per match this pass then computes what queryexec_ctx::prepare_match hands to consider(const matched_document &):
//   k_collect_count  one warp per match: lane j probes distinct term j of the query (does the term hold the document, and its freq);
//                    the lanes run the query's phrase nodes (phrase_match_count); every lane then runs the post-order collect program
//                    (planner.cpp plan_collect) over the presence bits into the matched-term mask, its popcount and the sum of its freqs
//   (scans)          terms and hits of the whole batch placed by the existing u32 -> u64 scan (launch_enc_scan): the result sizes are
//                    known before anything is written
//   k_collect_write  one warp per match, chunk by chunk of matches (each chunk's terms and hits go to device buffers sized for the chunk):
//                    lane j writes matched term j (its rank among the mask's bits), its freq and its hits with their payloads (HitWalker,
//                    hitcursor.h)
#pragma once

// query of global match m: the last q with q_offsets[q] <= m
__device__ __forceinline__ uint32_t collect_query_of(const uint64_t *q_offsets, uint32_t nq, uint64_t m) {
        uint32_t lo = 0, hi = nq; // q_offsets[lo] <= m < q_offsets[hi]
        while (hi - lo > 1u) {
                const uint32_t mid = (lo + hi) >> 1;
                if (q_offsets[mid] <= m)
                        lo = mid;
                else
                        hi = mid;
        }
        return lo;
}

// the post-order collect program over the presence bits of the query's terms and phrases: the matched-term mask of the root, which
// holds the document iff *has (queryexec_ctx.cpp:382-648; planner.cpp plan_collect has the rules)
__device__ uint32_t collect_eval(const CollectOp *prog, uint32_t nprog, const CollectPhrase *phrases, uint32_t present, uint32_t phmask, bool *has) {
        uint32_t stack[kCollectMaxStack];
        uint32_t holds = 0; // bit i: stack entry i holds the document
        uint32_t sp    = 0;
        for (uint32_t i = 0; i < nprog; ++i) {
                const CollectOp o = prog[i];
                uint32_t        m = 0;
                bool            h = false;
                if (o.kind == CO_TERM) {
                        h = o.arg != kEmptyTerm && ((present >> o.arg) & 1u);
                        m = h ? (1u << o.arg) : 0u;
                } else if (o.kind == CO_PHRASE) {
                        h = (phmask >> o.arg) & 1u;
                        m = h ? phrases[o.arg].mask : 0u;
                } else {
                        const uint32_t b = sp - o.nchildren;
                        if (o.kind == CO_NOT) { // required side only
                                h = ((holds >> b) & 1u) && !((holds >> (b + 1u)) & 1u);
                                m = stack[b];
                        } else if (o.kind == CO_OPTIONAL) { // main, plus opt where it holds the document
                                h = (holds >> b) & 1u;
                                m = stack[b] | (((holds >> (b + 1u)) & 1u) ? stack[b + 1u] : 0u);
                        } else { // AND: all children; OR / SOME: the children that hold the document
                                uint32_t cnt = 0;
                                for (uint32_t c = b; c < sp; ++c)
                                        if ((holds >> c) & 1u) {
                                                ++cnt;
                                                m |= stack[c];
                                        }
                                h = o.kind == CO_AND ? cnt == o.nchildren : o.kind == CO_OR ? cnt > 0u : cnt >= o.min;
                        }
                        sp = b;
                }
                if (!h)
                        m = 0;
                stack[sp] = m;
                holds     = (holds & ~(1u << sp)) | (uint32_t(h) << sp);
                ++sp;
        }
        *has = holds & 1u;
        return stack[0];
}

__global__ void __launch_bounds__(256) k_collect_count(const CollectParams P) {
        const uint64_t m    = P.m0 + (uint64_t(blockIdx.x) * 256u + threadIdx.x) / 32u;
        const uint32_t lane = threadIdx.x & 31u;
        if (m >= P.m1)
                return;
        const uint32_t     q = collect_query_of(P.q_offsets, P.nq, m);
        const uint32_t     d = P.docids[m];
        const CollectQuery Q = P.queries[q];
        const HitsView     hv = hits_view(P.ix);
        bool               found{false};
        uint32_t           freq{0};
        if (lane < Q.nterms)
                found = term_holds(hv, phrase_term(P.ix, P.terms[Q.term_begin + lane]), d, freq);
        const uint32_t present = __ballot_sync(0xffffffffu, found);
        bool           ph{false};
        if (lane < Q.nphrases) {
                const CollectPhrase F = P.phrases[Q.phrase_begin + lane];
                ph                    = phrase_match_count(P.ix, P.args + F.arg_begin, F.k, d) != 0u;
        }
        const uint32_t phmask = __ballot_sync(0xffffffffu, ph);
        bool           has{false};
        const uint32_t mask = collect_eval(P.prog + Q.prog_begin, Q.nprog, P.phrases + Q.phrase_begin, present, phmask, &has);
        uint32_t       hits = ((mask >> lane) & 1u) ? freq : 0u;
        for (int o = 16; o; o >>= 1)
                hits += __shfl_xor_sync(0xffffffffu, hits, o);
        if (lane == 0) {
                if (!has)
                        atomicOr(P.error, 1u);
                P.mask[m]   = mask;
                P.nterms[m] = uint32_t(__popc(mask));
                P.nhits[m]  = hits;
        }
}

__global__ void __launch_bounds__(256) k_collect_write(const CollectParams P) {
        const uint64_t m    = P.m0 + (uint64_t(blockIdx.x) * 256u + threadIdx.x) / 32u;
        const uint32_t lane = threadIdx.x & 31u;
        if (m >= P.m1)
                return;
        const uint32_t     q    = collect_query_of(P.q_offsets, P.nq, m);
        const uint32_t     d    = P.docids[m];
        const CollectQuery Q    = P.queries[q];
        const uint32_t     mask = P.mask[m];
        const bool         mine = (mask >> lane) & 1u;
        const HitsView     hv   = hits_view(P.ix);
        const uint64_t     t0   = P.term_scan[m], h0 = P.hit_scan[m]; // global
        if (lane == 0)
                P.term_offsets[m - P.m0] = t0;
        uint32_t   freq{0};
        PhraseTerm T;
        if (mine) {
                T = phrase_term(P.ix, P.terms[Q.term_begin + lane]);
                (void)term_holds(hv, T, d, freq);
        }
        uint32_t x = freq; // inclusive scan of the freqs over the lanes = hits of the matched terms before this one, in term order
        for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= uint32_t(o))
                        x += y;
        }
        if (!mine)
                return;
        const uint64_t t = t0 + uint32_t(__popc(mask & ((1u << lane) - 1u)));
        const uint64_t h = h0 + (x - freq);
        P.out_terms[t - P.term_base]   = P.terms[Q.term_begin + lane];
        P.out_freqs[t - P.term_base]   = freq;
        P.hit_offsets[t - P.term_base] = h;
        if (!freq)
                return;
        HitWalker w;
        w.init(hv, T, d);
        auto *out = reinterpret_cast<ulonglong2 *>(P.out_hits); // one 16-byte store per hit, trn_hit's padding zeroed
        for (uint64_t k = h - P.hit_base; w.c.left; ++k) {
                uint32_t       len;
                const uint32_t pos = w.next(len);
                out[k]             = make_ulonglong2(w.payload, (unsigned long long)(pos & 0xffffu) | ((unsigned long long)(len & 0xffu) << 16));
        }
}

cudaError_t launch_collect_count(const CollectParams &P, cudaStream_t stream) {
        const uint64_t n = P.m1 - P.m0;
        if (!n)
                return cudaSuccess;
        k_collect_count<<<unsigned((n + 7u) / 8u), 256, 0, stream>>>(P);
        return cudaGetLastError();
}

cudaError_t launch_collect_write(const CollectParams &P, cudaStream_t stream) {
        const uint64_t n = P.m1 - P.m0;
        if (!n)
                return cudaSuccess;
        k_collect_write<<<unsigned((n + 7u) / 8u), 256, 0, stream>>>(P);
        return cudaGetLastError();
}
