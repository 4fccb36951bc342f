// Percolator registry updates (trn_percolator_add / trn_percolator_remove, engine.cu; DESIGN.md §4): the term -> anchored-queries index,
// the unanchored list and the program storage are rebuilt on the device into new buffers, so that they hold what a fresh registration of
// every issued query would, minus the removed ones.  k_perc reads them unchanged.  Included by kernels.cu inside namespace trn.
//
//   keep         per old entry (a PercEntry of the index, or an id of the unanchored list): 1 unless its query is in the removed bitmap
//   (scan)       launch_enc_scan of the keep flags: the rank of every surviving entry
//   term counts  per term: its surviving old entries (the scan across its CSR range) plus its new entries (a binary search in the new
//                entries' sorted terms); scanned again into the new csr_off
//   scatter      thread = entry: a surviving old entry goes to its term's new start + its surviving rank inside the term, a new entry behind
//                the term's surviving old ones.  New ids are above every old one, so every term stays in ascending query id
//   programs     per issued id its ops / phrase terms / cover terms (0 for a removed query), scanned, then copied to the scanned offsets;
//                the phrase ops' term offsets are moved with their query's phrase terms
static constexpr int kPercUpdThreads = 256;

__device__ __forceinline__ uint32_t perc_upd_id(const PercEntry &e) {
        return e.query;
}
__device__ __forceinline__ uint32_t perc_upd_id(uint32_t q) {
        return q;
}
__device__ __forceinline__ bool perc_upd_removed(const uint32_t *removed, uint32_t q) {
        return removed && ((removed[q >> 5] >> (q & 31u)) & 1u);
}
// the first i in [0, n) with a[i] > v (n: none)
__device__ __forceinline__ uint64_t perc_upd_upper(const uint32_t *a, uint64_t n, uint32_t v) {
        uint64_t lo = 0, hi = n;
        while (lo < hi) {
                const uint64_t mid = (lo + hi) >> 1;
                if (a[mid] <= v)
                        lo = mid + 1;
                else
                        hi = mid;
        }
        return lo;
}
// the first i in [0, n) with a[i] >= v
__device__ __forceinline__ uint64_t perc_upd_lower(const uint32_t *a, uint64_t n, uint32_t v) {
        uint64_t lo = 0, hi = n;
        while (lo < hi) {
                const uint64_t mid = (lo + hi) >> 1;
                if (a[mid] < v)
                        lo = mid + 1;
                else
                        hi = mid;
        }
        return lo;
}

template <class T> __global__ void __launch_bounds__(kPercUpdThreads) k_perc_upd_keep(const T *in, uint64_t n, const uint32_t *removed, uint32_t *keep) {
        for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += uint64_t(gridDim.x) * blockDim.x)
                keep[i] = perc_upd_removed(removed, perc_upd_id(in[i])) ? 0u : 1u;
}

__global__ void __launch_bounds__(kPercUpdThreads) k_perc_upd_term_counts(const uint32_t *csr_off, uint32_t nterms, const unsigned long long *kscan,
                                                                          const uint32_t *new_terms, uint32_t nnew, uint32_t *cnt) {
        for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < nterms; t += gridDim.x * blockDim.x) {
                const uint64_t added = perc_upd_upper(new_terms, nnew, t) - perc_upd_lower(new_terms, nnew, t);
                cnt[t]               = uint32_t(kscan[csr_off[t + 1]] - kscan[csr_off[t]] + added);
        }
}

// threads [0, nold + nnew) place the entries, threads [0, nterms] write the new csr_off (the host checked that it fits 32 bits)
__global__ void __launch_bounds__(kPercUpdThreads) k_perc_upd_csr_scatter(const PercEntry *csr, const uint32_t *csr_off, uint32_t nterms, uint64_t nold,
                                                                          const uint32_t *keep, const unsigned long long *kscan, const PercEntry *new_e,
                                                                          const uint32_t *new_terms, uint32_t nnew, const unsigned long long *off,
                                                                          PercEntry *out, uint32_t *out_off) {
        const uint64_t n = max(nold + nnew, uint64_t(nterms) + 1u);
        for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += uint64_t(gridDim.x) * blockDim.x) {
                if (i <= nterms)
                        out_off[i] = uint32_t(off[i]);
                if (i < nold) {
                        if (!keep[i])
                                continue;
                        const uint32_t t = uint32_t(perc_upd_upper(csr_off, uint64_t(nterms) + 1u, uint32_t(i)) - 1u); // csr_off[t] <= i < csr_off[t + 1]
                        out[off[t] + (kscan[i] - kscan[csr_off[t]])] = csr[i];
                } else if (i < nold + nnew) {
                        const uint32_t j = uint32_t(i - nold), t = new_terms[j];
                        const uint64_t first = perc_upd_lower(new_terms, nnew, t);
                        out[off[t] + (kscan[csr_off[t + 1]] - kscan[csr_off[t]]) + (j - first)] = new_e[j];
                }
        }
}

// the surviving ids of the old unanchored list in order, then the new ones
__global__ void __launch_bounds__(kPercUpdThreads) k_perc_upd_unanch_scatter(const uint32_t *old, uint64_t nold, const uint32_t *keep,
                                                                             const unsigned long long *kscan, const uint32_t *add, uint32_t nadd, uint32_t *out) {
        for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nold + nadd; i += uint64_t(gridDim.x) * blockDim.x) {
                if (i < nold) {
                        if (keep[i])
                                out[kscan[i]] = old[i];
                } else
                        out[kscan[nold] + (i - nold)] = add[i - nold];
        }
}

// per issued id: its ops, phrase terms and cover terms, 0 for a removed query
__global__ void __launch_bounds__(kPercUpdThreads) k_perc_upd_prog_sizes(const PercQuery *queries, const PercOp *ops, uint32_t nq, const uint32_t *removed,
                                                                         uint32_t *nops, uint32_t *npt, uint32_t *ncov) {
        for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) {
                const bool      live = !perc_upd_removed(removed, q);
                const PercQuery Q    = queries[q];
                uint32_t        pt{0};
                if (live)
                        for (uint32_t i = 0; i < Q.nops; ++i) {
                                const PercOp o = ops[Q.op_begin + i];
                                if (o.op == PERC_PHRASE)
                                        pt += o.n;
                        }
                nops[q] = live ? Q.nops : 0u;
                npt[q]  = pt;
                ncov[q] = live ? Q.ncover : 0u;
        }
}

// thread = issued id: a live query's program, phrase terms and cover to the scanned offsets; a removed query becomes empty
__global__ void __launch_bounds__(kPercUpdThreads) k_perc_upd_prog_scatter(const PercQuery *queries, const PercOp *ops, const uint32_t *pterms,
                                                                           const uint32_t *covers, uint32_t nq, const uint32_t *removed,
                                                                           const unsigned long long *ops_at, const unsigned long long *pt_at,
                                                                           const unsigned long long *cov_at, PercQuery *out_q, PercOp *out_ops,
                                                                           uint32_t *out_pt, uint32_t *out_cov) {
        for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) {
                if (perc_upd_removed(removed, q)) {
                        out_q[q] = PercQuery{0, 0, 0, 0};
                        continue;
                }
                const PercQuery Q = queries[q];
                const uint32_t  ob = uint32_t(ops_at[q]), pb = uint32_t(pt_at[q]), cb = uint32_t(cov_at[q]);
                uint32_t        pt_old{0}, npt{0}; // the query's phrase terms are consecutive, in the order of its phrase ops
                for (uint32_t i = 0; i < Q.nops; ++i) {
                        PercOp o = ops[Q.op_begin + i];
                        if (o.op == PERC_PHRASE) {
                                if (!npt)
                                        pt_old = o.term;
                                o.term = pb + npt;
                                npt += o.n;
                        }
                        out_ops[ob + i] = o;
                }
                for (uint32_t k = 0; k < npt; ++k)
                        out_pt[pb + k] = pterms[pt_old + k];
                for (uint32_t k = 0; k < Q.ncover; ++k)
                        out_cov[cb + k] = covers[Q.cover_begin + k];
                out_q[q] = PercQuery{ob, Q.nops, cb, Q.ncover};
        }
}

static uint32_t perc_upd_grid(uint64_t n) {
        return uint32_t(std::max<uint64_t>(1, std::min<uint64_t>((n + kPercUpdThreads - 1) / kPercUpdThreads, 65535u * 4u)));
}

cudaError_t launch_perc_upd_keep(const PercEntry *csr, uint64_t n, const uint32_t *removed, uint32_t *keep, cudaStream_t stream) {
        if (n)
                k_perc_upd_keep<PercEntry><<<perc_upd_grid(n), kPercUpdThreads, 0, stream>>>(csr, n, removed, keep);
        return cudaGetLastError();
}

cudaError_t launch_perc_upd_keep(const uint32_t *ids, uint64_t n, const uint32_t *removed, uint32_t *keep, cudaStream_t stream) {
        if (n)
                k_perc_upd_keep<uint32_t><<<perc_upd_grid(n), kPercUpdThreads, 0, stream>>>(ids, n, removed, keep);
        return cudaGetLastError();
}

cudaError_t launch_perc_upd_csr(const PercEntry *csr, const uint32_t *csr_off, uint32_t nterms, uint64_t nold, const uint32_t *keep,
                                const unsigned long long *kscan, const PercEntry *new_e, const uint32_t *new_terms, uint32_t nnew, uint32_t *cnt,
                                unsigned long long *partials, unsigned long long *off, PercEntry *out, uint32_t *out_off, cudaStream_t stream) {
        if (nterms)
                k_perc_upd_term_counts<<<perc_upd_grid(nterms), kPercUpdThreads, 0, stream>>>(csr_off, nterms, kscan, new_terms, nnew, cnt);
        if (const cudaError_t e = launch_enc_scan(cnt, nterms, partials, off, stream); e != cudaSuccess)
                return e;
        const uint64_t n = std::max<uint64_t>(nold + nnew, uint64_t(nterms) + 1u);
        k_perc_upd_csr_scatter<<<perc_upd_grid(n), kPercUpdThreads, 0, stream>>>(csr, csr_off, nterms, nold, keep, kscan, new_e, new_terms, nnew, off, out,
                                                                                  out_off);
        return cudaGetLastError();
}

cudaError_t launch_perc_upd_unanch(const uint32_t *old, uint64_t nold, const uint32_t *keep, const unsigned long long *kscan, const uint32_t *add,
                                   uint32_t nadd, uint32_t *out, cudaStream_t stream) {
        if (nold + nadd)
                k_perc_upd_unanch_scatter<<<perc_upd_grid(nold + nadd), kPercUpdThreads, 0, stream>>>(old, nold, keep, kscan, add, nadd, out);
        return cudaGetLastError();
}

cudaError_t launch_perc_upd_prog_sizes(const PercQuery *queries, const PercOp *ops, uint32_t nq, const uint32_t *removed, uint32_t *nops, uint32_t *npt,
                                       uint32_t *ncov, cudaStream_t stream) {
        if (nq)
                k_perc_upd_prog_sizes<<<perc_upd_grid(nq), kPercUpdThreads, 0, stream>>>(queries, ops, nq, removed, nops, npt, ncov);
        return cudaGetLastError();
}

cudaError_t launch_perc_upd_prog_scatter(const PercQuery *queries, const PercOp *ops, const uint32_t *pterms, const uint32_t *covers, uint32_t nq,
                                         const uint32_t *removed, const unsigned long long *ops_at, const unsigned long long *pt_at,
                                         const unsigned long long *cov_at, PercQuery *out_q, PercOp *out_ops, uint32_t *out_pt, uint32_t *out_cov,
                                         cudaStream_t stream) {
        if (nq)
                k_perc_upd_prog_scatter<<<perc_upd_grid(nq), kPercUpdThreads, 0, stream>>>(queries, ops, pterms, covers, nq, removed, ops_at, pt_at, cov_at,
                                                                                           out_q, out_ops, out_pt, out_cov);
        return cudaGetLastError();
}
