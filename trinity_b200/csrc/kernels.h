// Launch wrappers implemented in kernels.cu
#pragma once
#include "device_types.h"
#include "hitcursor.h"
#include <cuda_runtime.h>

namespace trn {
uint32_t    exec_stage_bytes(int codec);
size_t      exec_smem_bytes(uint32_t tile_shift, uint32_t nslots, int mode, int codec);
int         exec_max_ctas_per_sm(uint32_t tile_shift, uint32_t nslots, int mode, int codec, bool filt = false); // filt: the filtered instantiations
cudaError_t launch_exec_tiles(const ExecParams &P, int grid, cudaStream_t stream);
uint32_t    exec_docs_stage_bytes();
uint32_t    exec_docs_cand_smem_bytes(bool with_membership); // per-warp shared memory of the candidate-driven path (membership bytes: trees with terms that are not necessary)
uint32_t    exec_docs_mixed_smem_bytes(); // per-warp shared memory of the mixed flat ANDs' run tickets (the candidate array, one gather buffer, counters)
size_t      exec_docs_smem_bytes(uint32_t exec_shift, uint32_t nslots, uint32_t stageBytes);
int         exec_docs_max_ctas_per_sm(uint32_t exec_shift, uint32_t nslots, uint32_t stageBytes, bool tree = false, bool lucene = false, bool filt = false);
cudaError_t launch_exec_docs(const ExecParams &P, int grid, cudaStream_t stream);
cudaError_t launch_query_scan(const unsigned long long *match_counts, uint32_t nq, uint64_t *q_offsets, cudaStream_t stream);
cudaError_t launch_item_scan(const DevQuery *queries, uint32_t nq, const uint32_t *item_cnt, const uint64_t *q_offsets, uint64_t *item_dst, cudaStream_t stream);
cudaError_t launch_gather(uint32_t total_items, const uint64_t *item_off, const uint32_t *item_cnt, const uint64_t *item_dst, const uint32_t *seg_docids,
                          const float *seg_scores, uint32_t *out_docids, float *out_scores, cudaStream_t stream);
cudaError_t launch_topk_select(const DevQuery *queries, uint32_t nq, const uint2 *cand, const uint32_t *cand_cursor, uint32_t k, uint32_t *out_docids,
                               float *out_scores, uint32_t *out_counts, cudaStream_t stream);
cudaError_t launch_topk_merge(const uint32_t *docids, const float *scores, uint32_t nshards, uint32_t nq, uint32_t k, uint32_t *out_docids, float *out_scores,
                              cudaStream_t stream);
size_t      score_flat_smem_bytes(uint32_t tile_shift, int threads);
uint32_t    score_flat_max_leaves();
cudaError_t launch_build_luts(const FlatLeaf *leaves, uint32_t nleaves, float *luts, cudaStream_t stream);
cudaError_t launch_score_flat(const ScoreParams &S, int threads, int num_sms, cudaStream_t stream);
cudaError_t launch_decode_stream(const DevIndex &ix, const DecUnit *units, const uint64_t *out_base, uint32_t total_units, uint32_t *docids, uint32_t *freqs,
                                 unsigned long long *sums, int num_sms, cudaStream_t stream);
cudaError_t launch_enc_scan(const uint32_t *in, uint64_t n, unsigned long long *partials, unsigned long long *out, cudaStream_t stream);
cudaError_t launch_enc_google_sizes(const EncParams &E, const EncPayloads &pay, cudaStream_t stream);
cudaError_t launch_enc_term_sizes(const EncParams &E, unsigned long long *chunk_bytes, cudaStream_t stream);
cudaError_t launch_enc_google_write(const EncParams &E, const EncPayloads &pay, cudaStream_t stream);
cudaError_t launch_enc_lucene_term_hits(const unsigned long long *term_begin, const unsigned long long *hit_begin, uint32_t nterms, unsigned long long *term_hits,
                                        cudaStream_t stream);
cudaError_t launch_enc_lucene_sizes(const EncLuceneParams &E, const EncPayloads &pay, cudaStream_t stream);
cudaError_t launch_enc_lucene_terms(const EncLuceneParams &E, const unsigned long long *fixed, unsigned long long *term_off, unsigned long long *hits_off,
                                    cudaStream_t stream);
cudaError_t launch_enc_lucene_write(const EncLuceneParams &E, const EncPayloads &pay, cudaStream_t stream);
cudaError_t launch_collect_count(const CollectParams &P, cudaStream_t stream); // the default exec mode's collect pass (collect.cuh)
cudaError_t launch_collect_write(const CollectParams &P, cudaStream_t stream);
uint32_t    kernel_max_k();
// query-token intersections (intersect.cuh): pass A (passb false) / pass B of trn_intersect, the dense copy of the distinct masks, the tiles' carries
size_t      isect_smem_bytes();
cudaError_t launch_isect(const IsectParams &P, bool lucene, bool passb, int num_sms, cudaStream_t stream);
cudaError_t launch_isect_compact(const IsectParams &P, uint64_t total_slots, const uint64_t *base, uint32_t *cursor, unsigned long long *out_mask, uint32_t *out_first,
                                 int num_sms, cudaStream_t stream);
cudaError_t launch_isect_carry(const IsectParams &P, unsigned long long *carry, cudaStream_t stream);
// percolator (percolate.cuh): the count (write false) and write passes of trn_percolate over one launch's documents
size_t      perc_smem_bytes(uint32_t max_len, uint32_t max_hash, bool write);
cudaError_t launch_perc(const PercParams &P, bool write, int num_sms, cudaStream_t stream);
// percolator registry updates (percolate_update.cuh): the keep flags of the old index / unanchored list, the index and unanchored rebuilds, and
// the program-storage compaction of trn_percolator_add / trn_percolator_remove
cudaError_t launch_perc_upd_keep(const PercEntry *csr, uint64_t n, const uint32_t *removed, uint32_t *keep, cudaStream_t stream);
cudaError_t launch_perc_upd_keep(const uint32_t *ids, uint64_t n, const uint32_t *removed, uint32_t *keep, cudaStream_t stream);
cudaError_t launch_perc_upd_csr(const PercEntry *csr, const uint32_t *csr_off, uint32_t nterms, uint64_t nold, const uint32_t *keep,
                                const unsigned long long *kscan, const PercEntry *new_e, const uint32_t *new_terms, uint32_t nnew, uint32_t *cnt,
                                unsigned long long *partials, unsigned long long *off, PercEntry *out, uint32_t *out_off, cudaStream_t stream);
cudaError_t launch_perc_upd_unanch(const uint32_t *old, uint64_t nold, const uint32_t *keep, const unsigned long long *kscan, const uint32_t *add,
                                   uint32_t nadd, uint32_t *out, cudaStream_t stream);
cudaError_t launch_perc_upd_prog_sizes(const PercQuery *queries, const PercOp *ops, uint32_t nq, const uint32_t *removed, uint32_t *nops, uint32_t *npt,
                                       uint32_t *ncov, cudaStream_t stream);
cudaError_t launch_perc_upd_prog_scatter(const PercQuery *queries, const PercOp *ops, const uint32_t *pterms, const uint32_t *covers, uint32_t nq,
                                         const uint32_t *removed, const unsigned long long *ops_at, const unsigned long long *pt_at,
                                         const unsigned long long *cov_at, PercQuery *out_q, PercOp *out_ops, uint32_t *out_pt, uint32_t *out_cov,
                                         cudaStream_t stream);
// indexer (index_docs.cuh): document ranks, sort keys, one pass of the keys-only radix sort, the postings pass of trn_index_documents
cudaError_t launch_index_doc_keys(const uint32_t *docids, uint32_t ndocs, unsigned long long *keys, cudaStream_t stream);
cudaError_t launch_index_doc_ranks(const unsigned long long *keys, uint32_t ndocs, uint32_t *rank_of, uint32_t *docid_of, unsigned long long *errors,
                                   cudaStream_t stream);
cudaError_t launch_index_keys(const IndexParams &P, cudaStream_t stream);
cudaError_t launch_radix_pass(const unsigned long long *in, unsigned long long *out, uint64_t n, uint32_t shift, uint32_t bits, uint32_t *counts,
                              unsigned long long *partials, unsigned long long *offsets, cudaStream_t stream, const uint32_t *vin = nullptr, uint32_t *vout = nullptr);
cudaError_t launch_post_flags(const unsigned long long *keys, uint64_t n, uint32_t *post_flag, uint32_t *term_flag, cudaStream_t stream);
cudaError_t launch_post_write(const IndexParams &P, const unsigned long long *keys, const uint32_t *ords, cudaStream_t stream);
cudaError_t launch_post_freqs(const IndexParams &P, uint64_t nposts, cudaStream_t stream);
cudaError_t launch_build_dense(const DevIndex &ix, const uint32_t *sel, const unsigned long long *blk_prefix, uint32_t nsel, uint64_t total_blocks,
                               uint32_t *dense, cudaStream_t stream);
// merge (merge.cuh): the device half of trn_merge_sources / trn_merge_sources_payloads
struct MergeList { // one participant list of an output term (lists of one term are consecutive, newest first)
        DevTerm  t;        // the term in its source's block directory
        uint32_t view;     // its source's entry in MergeParams::views
        uint32_t term;     // term index in that source (the hits directory's HitTerm)
        uint32_t cand;     // candidate (newest first): its registry masks d iff upd_first(d) < cand
        uint32_t rank;     // participant rank inside the term (0 = newest)
        uint32_t nparts;   // participants of the term
        uint32_t reencode; // 0: an appended chunk (decoded for docs_cnt only)
};
struct MergeParams {
        const HitsView *          views;
        const MergeList *         lists;
        uint32_t                  nlists;
        const unsigned long long *list_blk, *list_post; // nlists + 1 prefix sums of blocks / postings
        unsigned long long        nblocks, nposts;
        uint32_t *                docids, *freqs, *hcount; // decoded postings; hcount = freq of a re-encoded posting, else 0
        const unsigned long long *hoff;                    // scan of hcount
        uint32_t *                positions;
        uint8_t *                 plens;  // per decoded hit, only when a kept hit carries a payload and the call takes them: its length
        unsigned long long *      pays;   // and its payload, masked to the low plens[] bytes
        const uint32_t *          upd_docid, *upd_first;
        unsigned long long        nupd;
        uint32_t *                keep, *bitmap;
        const unsigned long long *kscan;
        uint32_t *                out_docids, *out_freqs, *out_positions;
        uint8_t *                 out_plens;  // plens / pays in the output order (with them only)
        unsigned long long *      out_pays;
        unsigned long long *      out_src;
        const unsigned long long *out_hoff;
        unsigned long long *      error; // first kept posting with [0] a payload hit, [1] a hit at position 0 without a payload or above 16383,
                                         // [2] a payload length above 8 (~0: none)
};
struct MergeCopy {
        const uint8_t *    src;
        unsigned long long dst, len;
        uint32_t           to_hits, header, hits_off; // header: a LUCENE index chunk whose first u32 becomes hits_off
};
cudaError_t launch_merge_decode(const MergeParams &P, cudaStream_t stream);
cudaError_t launch_merge_hits_decode(const MergeParams &P, bool payloads, cudaStream_t stream); // payloads: also fill plens / pays
cudaError_t launch_merge_keep(const MergeParams &P, cudaStream_t stream);
cudaError_t launch_merge_scatter(const MergeParams &P, cudaStream_t stream);
cudaError_t launch_merge_out_hits(const MergeParams &P, uint64_t nout, bool payloads, cudaStream_t stream); // payloads: also out_plens / out_pays
cudaError_t launch_merge_gather(const unsigned long long *a, const unsigned long long *idx, uint32_t n, unsigned long long *out, cudaStream_t stream);
cudaError_t launch_merge_popcount(const uint32_t *bitmap, uint64_t nwords, unsigned long long *count, cudaStream_t stream);
cudaError_t launch_merge_assemble(const MergeCopy *segs, uint32_t nsegs, uint8_t *index_out, uint8_t *hits_out, cudaStream_t stream);
} // namespace trn
